"""Where a tile of the wgmma tower spends its time: SM-clock phase stamps of net_tower_kernel (rz_net_tc.cu).

Builds the library with -DRZ_TOWER_STAMPS into a separate directory (the in-tree library is not touched), runs the ch5
tower on 32 768 random positions and prints, per phase, the cycles one tile spends there (math thread 0 of each CTA, and
the producer thread for the bar_empty waits), averaged over all tiles of the timed launches.  The card's name, power
limit and SM clock are read in the same run; the SM clock is also derived from the stamps and the launch time.

    python tools/tower_phases.py [--out DIR] [--n 32768] [--blocks 10] [--iters 5] [--cluster 2]
"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "reversi-alpha-zero_b200")
sys.path.insert(0, ROOT)
sys.path.insert(0, PKG)

# order of the kSt* enum in rz_net_tc.cu
PHASES = ["tiles", "tile", "k_loop", "wait_bar_full", "wait_wgmma", "wait_epi_bar", "epilogue_layer0", "epilogue_conv1",
          "epilogue_conv2", "epilogue_last", "head_features", "producer_wait_bar_empty"]


def build_stamped(out):
    """Build the library with the stamps under `out`: the sources are copied on every call (with their times, so make
    recompiles what changed); the in-tree objects, built without stamps, are copied once so that only the tower object
    has to be compiled."""
    src = os.path.join(PKG, "csrc")
    csrc = os.path.join(out, "reversi-alpha-zero_b200", "csrc")
    os.makedirs(csrc, exist_ok=True)
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(out, "include"), dirs_exist_ok=True)
    for f in os.listdir(src):
        first_object = f.endswith(".o") and f != "rz_net_tc.o" and not os.path.exists(os.path.join(csrc, f))
        if f.endswith((".cu", ".cuh")) or f == "Makefile" or first_object:
            shutil.copy2(os.path.join(src, f), csrc)
    subprocess.check_call(["make", "-C", csrc, "-j8", "DEFS=-DRZ_TOWER_STAMPS"], stdout=subprocess.DEVNULL)
    return os.path.join(csrc, "librz_engine.so")


def smi(fields):
    r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else f"unavailable ({r.stderr.strip()})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="build directory of the stamped library (default: a temporary directory)")
    ap.add_argument("--n", type=int, default=32768)
    ap.add_argument("--blocks", type=int, default=10)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--cluster", type=int, default=2, choices=[1, 2])
    ap.add_argument("--json", default=None, help="also write the result to this file")
    a = ap.parse_args()
    out = a.out or tempfile.mkdtemp(prefix="rz_stamps_")
    lib_path = build_stamped(out)

    from reversi_zero_b200 import _cabi
    _cabi.LIB_PATH = lib_path   # before anything loads the library
    import torch
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200 import net as N, device as D
    lib = _cabi.lib()
    lib.rz_tower_stamps.restype, lib.rz_tower_stamps.argtypes = C.c_int, [C.POINTER(C.c_ulonglong), C.c_int, C.c_int]
    assert lib.rz_tower_stamp_count() == len(PHASES), "PHASES out of step with the kernel's kSt* enum"

    N.set_tower_cluster(a.cluster)
    mc = M.ModelConfig(res_layer_num=a.blocks)
    net = N.Net(mc)
    net.load_weights(M.build_random_weights(mc, 0))
    rng = np.random.default_rng(0)
    x = rng.integers(0, 2 ** 64, size=a.n, dtype=np.uint64); r = rng.integers(0, 2 ** 64, size=a.n, dtype=np.uint64)
    d_own, d_en = D.to_device(x & r), D.to_device(x & ~r)
    d_pol, d_val = D.empty(a.n * 64, np.float32), D.empty(a.n, np.float32)
    s = torch.cuda.current_stream()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for _ in range(2):
        net.predict_dev(d_own, d_en, d_pol, d_val, a.n, N.IMPL_TCGEN05, D.stream_ptr(s))
    assert lib.rz_tower_stamps(None, sms, 1) == 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    clocks = []
    poll = threading.Thread(target=lambda: clocks.append(smi("clocks.sm")))
    e0.record(s)
    for _ in range(a.iters):
        net.predict_dev(d_own, d_en, d_pol, d_val, a.n, N.IMPL_TCGEN05, D.stream_ptr(s))
    e1.record(s)
    poll.start()   # while the launches run
    torch.cuda.synchronize()
    poll.join()
    ms = e0.elapsed_time(e1) / a.iters
    buf = (C.c_ulonglong * (sms * len(PHASES)))()
    assert lib.rz_tower_stamps(buf, sms, 1) == 0
    st = np.frombuffer(buf, dtype=np.uint64).reshape(sms, len(PHASES)).astype(np.float64)
    ctas = st[:, 0] > 0
    tiles = st[ctas, 0].sum()
    per_tile = {k: st[ctas, i].sum() / tiles for i, k in enumerate(PHASES) if i > 0}
    layers = 1 + 2 * a.blocks
    # least time the K loops can take: a CTA issues 2 warpgroups x 144 wgmma.m64n256k16 per 3x3 conv (2 x 2 for layer 0),
    # and an SM completes one every 128 cycles at the dense FP16 rate (4096 flop per cycle per SM: 989 TFLOP/s at
    # 1830 MHz over 132 SMs); the wait_* phases overlap MMAs already queued, so the K loop's stall is k_loop - floor
    floor = 128 * 2 * (144 * (layers - 1) + 2)
    # the busiest CTA's stamped time over the launch time gives the SM clock the kernel ran at
    busiest = st[ctas, 1].max() / a.iters
    res = dict(gpu=torch.cuda.get_device_name(), power_limit=smi("power.limit"), sm_clock_during_run=clocks[0] if clocks else None,
               sm_clock_from_stamps_mhz=round(busiest / (ms * 1e3), 1), n=a.n, res_blocks=a.blocks, cluster=a.cluster,
               ms_per_launch=round(ms, 3), ctas=int(ctas.sum()), tiles_per_launch=tiles / a.iters,
               kcycles_per_tile={k: round(v / 1e3, 1) for k, v in per_tile.items()},
               k_loop_mma_floor_kcycles=round(floor / 1e3, 1), k_loop_stall_kcycles=round((per_tile["k_loop"] - floor) / 1e3, 1),
               k_loop_share_of_mma_rate=round(floor / per_tile["k_loop"], 3))
    print(json.dumps(res))
    print(f"{res['gpu']}, power limit {res['power_limit']}, SM clock {res['sm_clock_during_run']} "
          f"({res['sm_clock_from_stamps_mhz']} MHz from stamps); n = {a.n}, {a.blocks} blocks, cluster {a.cluster}, "
          f"{ms:.2f} ms per launch")
    print(f"{'phase':28s} kcycles/tile")
    for k, v in per_tile.items():
        print(f"{k:28s} {v / 1e3:10.1f}")
    print(f"{'k_loop MMA floor':28s} {floor / 1e3:10.1f}   (k_loop at {floor / per_tile['k_loop']:.1%} of the MMA rate)")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    net.close()


if __name__ == "__main__":
    main()
