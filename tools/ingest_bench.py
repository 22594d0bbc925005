"""Trainer-side ingest microbenchmark (SURVEY 8(f).4): N play rows resident in HBM -> training arrays.
Algorithmic bytes per row: 280 read + 8 x (128 + 256 + 4) = 3104 written = 3384 B (outputs of 1M rows = 3.3 GB, far
beyond the 126 MB L2).  CUDA-event timing over back-to-back launches on the launching stream.  Also times the path
from a row FILE (read + H2D + kernel) and, as CPU baseline, what the reference trainer does with the equivalent JSON
file (json.load + the oracle restatement of convert_to_training_data) on a bounded sample.  Prints one JSON object."""
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "reversi-alpha-zero_b200"))


def synth_rows(n, seed=20260923):
    from reversi_zero_b200.worker import ingest as zi
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 2 ** 63, n, dtype=np.uint64)
    r = rng.integers(0, 2 ** 63, n, dtype=np.uint64)
    nv = (rng.integers(0, 60, (n, 64)) * (rng.integers(0, 4, (n, 64)) == 0)).astype(np.int32)
    nv[:, 19] += 1
    return zi.make_rows(a & r, a & ~r, nv, rng.integers(-1, 2, n).astype(np.int32))


def run(n=1 << 20, iters=20, warmup=3, cpu_rows=1024):
    import torch
    from reversi_zero_b200 import _cabi
    from reversi_zero_b200.worker import ingest as zi
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm = peaks.get("hbm_gbs", 3350.0)   # H100 SXM data-sheet HBM3 bandwidth when no measured peak is given
    rows = synth_rows(n)
    dev = torch.device("cuda", 0)
    d_rows = torch.from_numpy(rows.view(np.uint8).reshape(-1)).to(dev)
    states = torch.empty((8 * n, 2, 8, 8), dtype=torch.uint8, device=dev)
    policy = torch.empty((8 * n, 64), dtype=torch.float32, device=dev)
    z = torch.empty((8 * n,), dtype=torch.float32, device=dev)
    lib = _cabi.lib()
    s = torch.cuda.current_stream()

    def call():
        return lib.rz_ingest_dev(d_rows.data_ptr(), n, 1, 4, states.data_ptr(), policy.data_ptr(), z.data_ptr(), s.cuda_stream)
    for _ in range(warmup):
        _cabi.check(call(), "rz_ingest_dev")
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(iters):
        call()
    e1.record(s)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    bytes_per_row = 280 + 8 * (128 + 256 + 4)
    gbs = n * bytes_per_row / ms / 1e6
    res = dict(rows=n, records=8 * n, bytes_per_row=bytes_per_row, kernel_ms=ms, records_per_s=8 * n / ms * 1e3, gbs=gbs, hbm_peak_gbs=hbm,
               frac_of_measured_hbm=gbs / hbm)
    # from a row file on disk to device tensors (what a device-side trainer calls): file read + H2D of the rows + kernel
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "play_bench.rzrows")
        with open(path, "wb") as f:
            hd = np.zeros(1, np.dtype([("magic", "S8"), ("tau1", "<i4"), ("ctt", "<i4"), ("n", "<u8"), ("zero", "<u8")]))
            hd["magic"], hd["tau1"], hd["ctt"], hd["n"] = b"RZROWS\x00\x01", 1, 4, n
            f.write(hd.tobytes()); f.write(rows.tobytes())
        for _ in range(2):
            torch.cuda.synchronize(); t0 = time.perf_counter()
            r2, tau1, ctt = zi.read_play_rows(path)
            out = zi.to_training_tensors(r2, tau1, ctt, 0)
            torch.cuda.synchronize(); dt = time.perf_counter() - t0
        assert torch.equal(out[0], states) and torch.equal(out[1], policy)
        res["from_file_s"] = dt
        res["from_file_records_per_s"] = 8 * n / dt
    # CPU baseline: the reference trainer's way on the same kind of data, bounded sample
    from oracle import ingest as oi
    sub = rows[:cpu_rows]
    es, ep, ez = oi.rows_to_training_arrays(sub["own"], sub["enemy"], sub["n_visit"], sub["z"], 1, 4)
    recs = [[[int(a[0].reshape(-1).dot(1 << np.arange(64, dtype=object))), int(a[1].reshape(-1).dot(1 << np.arange(64, dtype=object)))],
             [float(v) for v in p], int(zz)] for a, p, zz in zip(es, ep, ez)]
    with tempfile.TemporaryDirectory() as d:
        jp = os.path.join(d, "play_bench.json")
        with open(jp, "wt") as f:
            json.dump(recs, f)
        json_bytes = os.path.getsize(jp)
        from oracle import bitboard as ob
        t0 = time.perf_counter()
        data = json.load(open(jp, "rt"))
        sl, pl, zl = [], [], []
        for state, pol, zz in data:  # worker/optimize.py:215-231
            sl.append([ob.bit_to_array(state[0], 64).reshape(8, 8), ob.bit_to_array(state[1], 64).reshape(8, 8)])
            pl.append(pol); zl.append(zz)
        a_s, a_p, a_z = np.array(sl), np.array(pl), np.array(zl)
        dt = time.perf_counter() - t0
    assert np.array_equal(a_s, es) and np.array_equal(a_p, ep)
    res["cpu_baseline"] = dict(kind="port", cores=1, sample="%d rows = %d records, %.1f MB of JSON: json.load + convert_to_training_data loop" % (
        cpu_rows, 8 * cpu_rows, json_bytes / 1e6), records_per_s=8 * cpu_rows / dt, json_bytes_per_record=json_bytes / (8 * cpu_rows))
    return res


if __name__ == "__main__":
    print(json.dumps(run(*(int(a) for a in sys.argv[1:]))))
