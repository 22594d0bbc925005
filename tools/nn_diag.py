"""Numerics diagnostic for the wgmma tower (DESIGN.md section 5, tests/test_net_gpu.py): for three kinds of weights --
`--new` random-init (the north-star configuration), randomly perturbed BatchNorm statistics (the r1 stress case), and
trained-like weights (BatchNorm statistics calibrated to each layer's own pre-activation, random gamma / beta / biases) --
and towers of 0..10 residual blocks (the same leading weights, so the rows are the error after each depth), it prints

    kernel vs fp32 reference        what a user of the reference's Keras forward would see
    fp16-operand model vs fp32      what the NUMBER FORMAT costs (oracle/nn.py forward_fp16_operands: operands rounded to
                                    fp16, everything else exact) -- the floor of any single-pass fp16 tensor-core evaluation
    kernel vs fp16-operand model    what the KERNEL adds on top (accumulation order / tensor-core accumulator rounding)

for the tower output, the policy logits and the value logit.  `python tools/nn_diag.py [OUT.json]` also writes the rows
to OUT.json."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "reversi-alpha-zero_b200"))


def weights_of(kind, mc, seed, planes_cal):
    from oracle import nn as onn
    from reversi_zero_b200.agent import model as M
    if kind == "random-init":
        return M.build_random_weights(mc, seed)
    w = M.build_random_weights(mc, seed, perturb_bn=True)
    if kind == "calibrated":
        onn.calibrate_bn(w, planes_cal, mc.res_layer_num)
    return w


def main():
    import torch
    from oracle import nn as onn
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200 import net as N, device as D
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_net_gpu import selfplay_positions
    n = 64
    own, enemy = selfplay_positions(n, 5)
    planes = onn.planes_from_bitboards(own, enemy)
    own_c, enemy_c = selfplay_positions(256, 11)
    planes_cal = onn.planes_from_bitboards(own_c, enemy_c)
    d_own, d_en = D.to_device(own), D.to_device(enemy)
    rows = []
    for kind in ("random-init", "perturbed", "calibrated"):
        for R in (0, 1, 2, 4, 6, 8, 10):
            mc = M.ModelConfig(cnn_filter_num=256, res_layer_num=R, value_fc_size=256)
            w = weights_of(kind, mc, 5, planes_cal)
            net = N.Net(mc)
            net.load_weights(w)
            d_pol, d_val, d_tow = D.empty(n * 64, np.float32), D.empty(n, np.float32), D.empty(n * 64 * 256, np.float32)
            d_log, d_vl = D.empty(n * 64, np.float32), D.empty(n, np.float32)
            net.debug_heads_dev(d_own, d_en, d_pol, d_val, d_log, d_vl, n, tower_t=d_tow)
            torch.cuda.synchronize()
            got = dict(tower=d_tow.cpu().numpy().reshape(n, 64, 256).transpose(0, 2, 1).reshape(n, 256, 8, 8),
                       logits=d_log.cpu().numpy().reshape(n, 64), vlogit=d_vl.cpu().numpy(), policy=d_pol.cpu().numpy().reshape(n, 64),
                       value=d_val.cpu().numpy())
            net.close()
            ref = dict(zip(("policy", "value", "logits", "vlogit", "tower"), onn.forward_logits(w, planes, R)))
            emu = dict(zip(("policy", "value", "logits", "vlogit", "tower"), onn.forward_fp16_operands(w, planes, R)))
            row = dict(weights=kind, res_blocks=R, tower_rms=float(np.sqrt((ref["tower"] ** 2).mean())), tower_absmax=float(np.abs(ref["tower"]).max()),
                       logits_absmax=float(np.abs(ref["logits"]).max()), vlogit_absmax=float(np.abs(ref["vlogit"]).max()))
            for k in ("tower", "logits", "vlogit", "policy", "value"):
                row[f"{k}_kernel_vs_fp32"] = float(np.abs(got[k] - ref[k]).max())
                row[f"{k}_format_vs_fp32"] = float(np.abs(emu[k] - ref[k]).max())
                row[f"{k}_kernel_vs_format"] = float(np.abs(got[k] - emu[k]).max())
            rows.append(row)
            print(f"{kind:11s} R={R:2d} tower rms {row['tower_rms']:.3g} | tower: kernel {row['tower_kernel_vs_fp32']:.3g} format {row['tower_format_vs_fp32']:.3g} "
                  f"kernel-format {row['tower_kernel_vs_format']:.3g} | logits: {row['logits_kernel_vs_fp32']:.3g} / {row['logits_format_vs_fp32']:.3g} / "
                  f"{row['logits_kernel_vs_format']:.3g} | vlogit: {row['vlogit_kernel_vs_fp32']:.3g} / {row['vlogit_format_vs_fp32']:.3g} / "
                  f"{row['vlogit_kernel_vs_format']:.3g}", flush=True)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(dict(positions=n, gpu=torch.cuda.get_device_name(), columns="max-abs errors; kernel = wgmma tower, "
                           "format = fp16-operand model, fp32 = reference", rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
