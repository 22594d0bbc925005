"""Model loading for interactive play (reference play_game/common.py)."""
from logging import getLogger

import numpy as np

from ..worker.self_play import weight_source_path, keras_h5_source_path

logger = getLogger(__name__)


def model_source_path(config):
    """play_game/common.py:5-14: the newest next-generation weights or the best weights, in the order
    ``play.use_newest_next_generation_model`` gives.  Unlike self-play, nothing is random-initialised: with neither
    there the engine has nothing to play with."""
    path = weight_source_path(config)
    if path is not None:
        return path
    h5_path = keras_h5_source_path(config)
    if h5_path is not None:
        raise RuntimeError(f"{h5_path} exists but its engine-side twin (*.rzblob.npy) does not: run "
                           f"`python tools/export_keras_weights.py <model_config.json> {h5_path}` on the trainer side "
                           f"(INTEGRATION.md section 4)")
    raise RuntimeError("No models found!")


def load_model(config, device=0):
    from ..net import Net
    path = model_source_path(config)
    net = Net(config.model, device)
    net.load_blob(np.load(path))
    logger.info(f"loaded weights from {path}")
    return net
