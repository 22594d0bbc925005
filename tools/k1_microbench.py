"""K1 microbenchmark (BASELINE.json config 5): 10M positions resident in HBM, CUDA-event timing over
back-to-back launches; inputs (160 MB + outputs) exceed the 126 MB L2.  Prints one JSON object."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "reversi-alpha-zero_b200"))


def d_out_check(lib, D, d_own, d_enemy, n):
    import numpy as np
    out = D.empty(n, np.uint64)
    lib.rz_find_correct_moves_dev(D.ptr(d_own), D.ptr(d_enemy), D.ptr(out), n, D.stream_ptr())
    import torch
    torch.cuda.synchronize()
    return out


def run(n=10_000_000, iters=100, warmup=5, with_cpu=True):
    import torch
    from reversi_zero_b200 import _cabi, device as D
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm = peaks.get("hbm_gbs", 3350.0)   # H100 SXM data-sheet HBM3 bandwidth when no measured peak is given
    rng = np.random.default_rng(20260922)
    a = rng.integers(0, 2 ** 64, size=n, dtype=np.uint64)
    b = rng.integers(0, 2 ** 64, size=n, dtype=np.uint64)
    r = rng.integers(0, 2 ** 64, size=n, dtype=np.uint64)
    own, enemy = a & r, a & ~r
    pos = rng.integers(0, 64, size=n, dtype=np.uint8)
    d_own, d_enemy, d_pos = D.to_device(own), D.to_device(enemy), D.to_device(pos)
    d_out = D.empty(n, np.uint64)
    lib = _cabi.lib()
    s = torch.cuda.current_stream()
    res = {}
    for name, bytes_per, call in (
        ("find_correct_moves", 24, lambda: lib.rz_find_correct_moves_dev(D.ptr(d_own), D.ptr(d_enemy), D.ptr(d_out), n, D.stream_ptr(s))),
        ("calc_flip", 25, lambda: lib.rz_calc_flip_dev(D.ptr(d_pos), D.ptr(d_own), D.ptr(d_enemy), D.ptr(d_out), n, D.stream_ptr(s))),
    ):
        for _ in range(warmup):
            _cabi.check(call(), name)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for _ in range(iters):
            call()
        e1.record(s)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        gbs = n * bytes_per / ms / 1e6
        res[name] = dict(ms=ms, gpos_per_s=n / ms / 1e6, gbs=gbs, frac_of_measured_hbm=gbs / hbm, bytes_per_position=bytes_per)
    # fused environment step (rz_step_dev, env/reversi_env.py:42-85) on reachable-looking positions: every env plays pos if it
    # is legal for black, else its lowest legal move (algorithmic bytes per SURVEY 8(d): 17 in + 25 out = 42 B / position)
    legal = D.to_numpy_u64(d_out_check(lib, D, d_own, d_enemy, n))
    low = (legal & (~legal + np.uint64(1)))
    act = np.where(legal != 0, np.log2(np.maximum(low, 1).astype(np.float64)).astype(np.int8), np.int8(0)).astype(np.int8)
    st = dict(black=D.to_device(own), white=D.to_device(enemy), nxt=D.to_device(np.ones(n, np.uint8)), turn=D.to_device(np.zeros(n, np.uint8)),
              done=D.to_device(np.zeros(n, np.uint8)), win=D.to_device(np.zeros(n, np.uint8)), act=D.to_device(act), legal=D.empty(n, np.uint64))
    call = lambda: lib.rz_step_dev(D.ptr(st["black"]), D.ptr(st["white"]), D.ptr(st["nxt"]), D.ptr(st["turn"]), D.ptr(st["done"]),
                                   D.ptr(st["win"]), D.ptr(st["act"]), D.ptr(st["legal"]), n, D.stream_ptr(s))
    master = {k: st[k].clone() for k in ("black", "white", "nxt", "turn", "done", "win")}
    total = 0.0
    reps = 12
    for it in range(reps + 2):
        for k, v in master.items():       # every timed launch steps the SAME fresh states (restored outside the timed region)
            st[k].copy_(v)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        _cabi.check(call(), "rz_step_dev")
        e1.record(s)
        torch.cuda.synchronize()
        if it >= 2:
            total += e0.elapsed_time(e1)
    ms = total / reps
    res["step"] = dict(ms=ms, gpos_per_s=n / ms / 1e6, gbs=n * 42 / ms / 1e6, frac_of_measured_hbm=n * 42 / ms / 1e6 / hbm, bytes_per_position=42,
                       note="single launches on fresh states (black to move, a legal move each), events around each launch")
    res["n"] = n
    res["hbm_peak_gbs"] = hbm
    if not with_cpu:
        return res
    # CPU oracle on one core for scale
    from oracle import bitboard as ob
    t = time.time(); ob.find_correct_moves_batch(own[:2_000_000], enemy[:2_000_000]); dt = time.time() - t
    res["cpu_oracle_find_correct_moves_mpos_per_s_1core"] = 2.0 / dt
    # the reference's own compiled Cython (oracle/_ref, built from lib/alt/bitboard_cython.pyx) on one core
    from oracle import ref_native
    if ref_native.available():
        bb, _ = ref_native.load()
        m = 500_000
        t = time.time()
        ref = np.fromiter((bb.find_correct_moves(int(o), int(e)) for o, e in zip(own[:m], enemy[:m])), dtype=np.uint64, count=m)
        dt = time.time() - t
        res["cpu_reference_cython_find_correct_moves_mpos_per_s_1core"] = m / dt / 1e6
        res["cpu_reference_matches_first_500k"] = bool(np.array_equal(ref, D.to_numpy_u64(d_out_check(lib, D, d_own, d_enemy, n))[:m]))
    res["n"] = n
    res["hbm_peak_gbs"] = hbm
    return res


if __name__ == "__main__":
    # the default formulation (bit-sliced, inputs staged through shared memory) in this process; the others (RZ_K1_IMPL is
    # read once per process) in children: "bitsliced" = the same arithmetic without staging, "scalar" = the round-1 kernels
    res = run()
    res["impl"] = os.environ.get("RZ_K1_IMPL", "staged (default)")
    if "--both" in sys.argv and "RZ_K1_IMPL" not in os.environ:
        import subprocess
        for impl in ("bitsliced", "scalar"):
            out = subprocess.run([sys.executable, os.path.abspath(__file__)], env=dict(os.environ, RZ_K1_IMPL=impl), capture_output=True, text=True)
            try:
                sc = json.loads(out.stdout.strip().splitlines()[-1])
                res[impl + "_formulation"] = {k: sc[k] for k in ("find_correct_moves", "calc_flip")}
            except Exception as ex:
                res[impl + "_formulation"] = dict(error=str(ex), stderr=out.stderr[-500:])
    print(json.dumps(res))
