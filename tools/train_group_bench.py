"""Data-parallel training step of the ch5 network (rz_trainer_create_group) against the plain one-device trainer: for each
trainer and global batch, ms per step from CUDA events on the primary after warm-up, records/s, and the host time to
enqueue one step on an idle device (the least of 5; the step returns before the devices finish).  The GPU name and power
limit are read in the same run.

With one GPU visible it alternates the plain trainer and the group [0] `--repeats` times and times [0, 0] and
[0] * 8 (replicas sharing one device: what the exchanges and the enqueue cost); with more GPUs it also runs groups of
1, 2, 4 and 8 distinct devices (as many as are visible).  One JSON line per measurement.

    python tools/train_group_bench.py [--batches 256 1024 2048] [--steps 20] [--warmup 3] [--repeats 3] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "reversi-alpha-zero_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from train_bench import gpu_info  # noqa: E402


def dataset(n_records=65536):
    import torch
    g = torch.Generator(device="cuda:0").manual_seed(0)
    states = (torch.rand((n_records, 2, 8, 8), generator=g, device="cuda:0") < 0.3).to(torch.uint8)
    policy = torch.rand((n_records, 64), generator=g, device="cuda:0")
    policy /= policy.sum(dim=1, keepdim=True)
    z = torch.randint(-1, 2, (n_records,), generator=g, device="cuda:0").float()
    perm = torch.randperm(n_records, generator=g, device="cuda:0").to(torch.int32)
    return (states, policy, z), perm


def run(devices, batch, steps, warmup, data, perm):
    """devices None: the plain trainer"""
    import torch
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200 import train as T
    mc = M.ModelConfig()  # ch5: 256 filters, 10 residual blocks, value_fc 256
    n = perm.numel()
    tr = T.Trainer(mc, max_batch=batch, devices=devices)
    tr.load_blob(M.weights_to_blob(mc, M.build_random_weights(mc, 0)))
    ids = [perm[(k * batch) % (n - batch):][:batch].contiguous() for k in range(warmup + steps)]
    for k in range(warmup):
        tr.step(*data, ids[k], 0.01)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(warmup, warmup + steps):
        loss = tr.step(*data, ids[k], 0.01)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    # enqueue time on an idle device: back to back, a full launch queue would make the host wait for the device
    enqueue = []
    for k in range(warmup, warmup + min(steps, 5)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tr.step(*data, ids[k], 0.01)
        enqueue.append(time.perf_counter() - t0)
    torch.cuda.synchronize()
    tr.close()
    return dict(config="ch5", trainer="plain" if devices is None else "group", devices=devices, batch=batch, steps=steps,
                ms_per_step=ms, records_per_s=batch / ms * 1e3, host_enqueue_ms_per_step=min(enqueue) * 1e3,
                final_loss=[float(x) for x in loss.cpu()])


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[256, 1024, 2048])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    info = gpu_info()
    data, perm = dataset()
    n_gpus = torch.cuda.device_count()
    plan = []
    for b in a.batches:
        for rep in range(a.repeats):   # plain and group-of-one alternated, for the spread between repeats
            plan += [(None, b, rep), ([0], b, rep)]
        plan += [([0, 0], b, 0), ([0] * 8, b, 0)]
        plan += [(list(range(k)), b, 0) for k in (2, 4, 8) if k <= n_gpus]
    lines = []
    for devices, b, rep in plan:
        line = json.dumps({**info, "visible_gpus": n_gpus, "repeat": rep, **run(devices, b, a.steps, a.warmup, data, perm)})
        print(line, flush=True)
        lines.append(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
