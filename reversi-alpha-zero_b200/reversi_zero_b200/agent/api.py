"""Mirror of the reference's ``ReversiModelAPI`` (agent/api.py:20-45): ``predict(x)`` with
``x`` = ``(2,8,8)`` or ``(N,2,8,8)`` planes ``[own, enemy]`` of the side to move, returning
``(policy (64,)|(N,64), value (1,)|(N,1))`` -- evaluated by the CUDA network (wgmma tower for the
256-filter model).  The multi-process pipe server of the reference (agent/api.py:48-141) has no
equivalent: batching happens on the device inside the engine."""
import numpy as np

from ..net import Net, IMPL_AUTO


class ReversiModelAPI:
    def __init__(self, config, agent_model, impl=IMPL_AUTO):
        """agent_model: a ``reversi_zero_b200.net.Net`` (or any object with ``predict_planes``)."""
        self.config = config
        self.agent_model = agent_model
        self.impl = impl

    def predict(self, x):
        x = np.asarray(x)
        assert x.ndim in (3, 4)
        assert x.shape == (2, 8, 8) or x.shape[1:] == (2, 8, 8)
        orig_ndim = x.ndim
        if x.ndim == 3:
            x = x.reshape(1, 2, 8, 8)
        policy, value = self._do_predict(x)
        if orig_ndim == 3:
            return policy[0], value[0]
        return policy, value

    def _do_predict(self, x):
        policy, value = self.agent_model.predict_planes(x, self.impl)
        return policy, value.reshape(-1, 1)
