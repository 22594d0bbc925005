"""Play-JSON ingest on the device (rz_ingest_json_dev) against the reference trainer's CPU path; prints one JSON line.

    python tools/json_ingest_bench.py [--records 1048576] [--iters 10] [--cpu-sample 20000]

  * device: CUDA events around rz_ingest_json_dev on a text of --records records already in device memory, outputs
    preallocated (index pass, the record-count read, parse pass) -> GB/s of JSON text and records/s
  * file: wall time of worker.ingest.read_play_json on the same text written to a temporary file (read, H2D, parse)
  * cpu: json.loads + the reference's convert_to_training_data loop (worker/optimize.py:215-231) on --cpu-sample records
  * the card's name and power limit, read in the same run
The text is engine-like: 4096 distinct records (visit fractions n/total in repr form, one-hot policies, z = +-1)
repeated to the requested count.
"""
import argparse
import ctypes as C
import json
import os
import random
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "reversi-alpha-zero_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402


def make_records(n_distinct, seed=0):
    rng = random.Random(seed)
    recs = []
    for i in range(n_distinct):
        occ = rng.getrandbits(64)
        own = occ & rng.getrandbits(64)
        if i % 4 == 3:  # tau-0: one-hot
            pol = [0.0] * 64
            pol[rng.randrange(64)] = 1.0
        else:
            n = [rng.randrange(0, 60) if rng.random() < 0.3 else 0 for _ in range(64)]
            n[rng.randrange(64)] += 1
            tot = sum(n)
            pol = [x / tot for x in n]
        recs.append([[own, occ & ~own], pol, 1 if i % 2 else -1])
    return recs


def card():
    import torch
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True)
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=out.stdout.strip() if out.returncode == 0 else None)


def cpu_baseline(text):
    """json.load + OptimizeWorker.convert_to_training_data (worker/optimize.py:215-231) restated"""
    from oracle.bitboard import bit_to_array
    t0 = time.perf_counter()
    data = json.loads(text)
    state_list, policy_list, z_list = [], [], []
    for state, policy, z in data:
        own, enemy = bit_to_array(state[0], 64).reshape((8, 8)), bit_to_array(state[1], 64).reshape((8, 8))
        state_list.append([own, enemy])
        policy_list.append(policy)
        z_list.append(z)
    np.array(state_list), np.array(policy_list), np.array(z_list)
    return time.perf_counter() - t0, len(data)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1 << 20)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--cpu-sample", type=int, default=20000)
    a = ap.parse_args()
    import torch
    from reversi_zero_b200 import _cabi
    from reversi_zero_b200.worker import ingest as I
    assert torch.cuda.is_available(), "the device ingest needs a CUDA device"
    recs = make_records(4096)
    body = ", ".join(json.dumps(r) for r in recs)
    reps = -(-a.records // len(recs))
    text = ("[" + ", ".join([body] * reps) + "]").encode()
    n_rec = reps * len(recs)
    dev = torch.device("cuda", 0)
    d_text = torch.frombuffer(bytearray(text), dtype=torch.uint8).to(dev)
    states = torch.empty((n_rec, 2, 8, 8), dtype=torch.uint8, device=dev)
    policy = torch.empty((n_rec, 64), dtype=torch.float32, device=dev)
    z = torch.empty((n_rec,), dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream()
    nr, off = C.c_size_t(), C.c_size_t()

    def run():
        _cabi.check(_cabi.lib().rz_ingest_json_dev(d_text.data_ptr(), len(text), n_rec, states.data_ptr(), policy.data_ptr(),
                                                    z.data_ptr(), C.byref(nr), C.byref(off), stream.cuda_stream), "rz_ingest_json_dev")

    run()
    run()
    assert nr.value == n_rec
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(a.iters):
        ev0.record(stream)
        run()
        ev1.record(stream)
        ev1.synchronize()
        times.append(ev0.elapsed_time(ev1) / 1e3)
    t_dev = float(np.median(times))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "play_bench.json")
        with open(path, "wb") as f:
            f.write(text)
        I.read_play_json(path)
        torch.cuda.synchronize()
        walls = []
        for _ in range(3):
            t0 = time.perf_counter()
            I.read_play_json(path)
            torch.cuda.synchronize()
            walls.append(time.perf_counter() - t0)
    sample = ("[" + ", ".join(json.dumps(r) for r in (recs * (-(-a.cpu_sample // len(recs))))[:a.cpu_sample]) + "]")
    t_cpu, n_cpu = cpu_baseline(sample)
    print(json.dumps(dict(
        metric="json_ingest", records=n_rec, text_bytes=len(text), bytes_per_record=round(len(text) / n_rec, 1),
        device_call_s=round(t_dev, 5), device_call_spread_s=[round(min(times), 5), round(max(times), 5)],
        device_gb_per_s=round(len(text) / t_dev / 1e9, 2), device_records_per_s=round(n_rec / t_dev),
        file_to_tensors_s=round(float(np.median(walls)), 4), file_records_per_s=round(n_rec / float(np.median(walls))),
        cpu_records=n_cpu, cpu_s=round(t_cpu, 4), cpu_records_per_s=round(n_cpu / t_cpu), **card())))


if __name__ == "__main__":
    main()
