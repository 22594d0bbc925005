"""What one training step of the ch5 network puts on the device, for comparing two builds of the library: per stream,
the ordered (kernel name, grid, block) of one step and its memcpy / memset counts, from torch.profiler's CUDA activities
after warm-up; and the device memory a trainer takes at each `--max-batches` (cudaMemGetInfo around its creation; other
processes on the device move that number, so read it on a quiet device or repeat it).  Every step of the traced window
must launch the same sequence.

    python tools/train_launch_trace.py --out new.json [--lib OTHER/librz_engine.so] [--devices 0 0] [--batch 256]
    python tools/train_launch_trace.py --compare old.json new.json     # exit status 1 when they differ
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "reversi-alpha-zero_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def memory_taken(mc, devices, max_batch):
    import torch
    from reversi_zero_b200 import train as T
    torch.cuda.synchronize()
    before = torch.cuda.mem_get_info(0)[0]
    tr = T.Trainer(mc, max_batch=max_batch, devices=devices)
    taken = before - torch.cuda.mem_get_info(0)[0]
    tr.close()
    return taken


def trace(mc, devices, batch, steps, warmup):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200 import train as T
    from train_group_bench import dataset
    data, perm = dataset()
    tr = T.Trainer(mc, max_batch=batch, devices=devices)
    tr.load_blob(M.weights_to_blob(mc, M.build_random_weights(mc, 0)))
    ids = [perm[k * batch:][:batch].contiguous() for k in range(warmup + steps)]
    for k in range(warmup):
        tr.step(*data, ids[k], 0.01)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(warmup, warmup + steps):
            tr.step(*data, ids[k], 0.01)
        torch.cuda.synchronize()
    tr.close()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    streams = {}
    for e in sorted((e for e in events if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")), key=lambda e: e["ts"]):
        a = e["args"]
        streams.setdefault(a["stream"], []).append([e["name"], a["grid"], a["block"]] if e["cat"] == "kernel" else [e["cat"]])
    per_stream = []
    for seq in streams.values():
        assert len(seq) % steps == 0, f"{len(seq)} device operations on one stream in {steps} steps"
        one = seq[:len(seq) // steps]
        assert seq == one * steps, "the steps of the window differ in what they launch"
        per_stream.append(dict(kernels=[op for op in one if len(op) == 3], memcpy=one.count(["gpu_memcpy"]),
                               memset=one.count(["gpu_memset"])))
    return sorted(per_stream, key=lambda s: json.dumps(s))


def compare(path_a, path_b):
    a, b = (json.load(open(p)) for p in (path_a, path_b))
    same = True
    for key in sorted(set(a) | set(b)):
        if key in ("lib", "gpu", "power_limit", "max_sm_clock"):
            continue
        eq = a.get(key) == b.get(key)
        same &= eq
        if key == "streams":
            print(f"streams: {'equal' if eq else 'DIFFERENT'}; per stream (kernels, memcpy, memset) per step: "
                  f"{[(len(s['kernels']), s['memcpy'], s['memset']) for s in a[key]]} vs "
                  f"{[(len(s['kernels']), s['memcpy'], s['memset']) for s in b[key]]}")
            for sa, sb in zip(a[key], b[key]):
                for i, (ka, kb) in enumerate(zip(sa["kernels"], sb["kernels"])):
                    if ka != kb:
                        print(f"  first difference at kernel {i}: {ka} vs {kb}")
                        break
        else:
            print(f"{key}: {'equal' if eq else 'DIFFERENT'}: {a.get(key)} vs {b.get(key)}")
    return same


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="trace this build of librz_engine.so instead of the tree's")
    ap.add_argument("--devices", type=int, nargs="+", default=None, help="a data-parallel group; default: the plain trainer")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--max-batches", type=int, nargs="*", default=[256, 2048])
    ap.add_argument("--out", default=None)
    ap.add_argument("--compare", nargs=2, metavar="JSON", default=None)
    a = ap.parse_args()
    if a.compare:
        sys.exit(0 if compare(*a.compare) else 1)
    from reversi_zero_b200 import _cabi
    if a.lib:
        _cabi.LIB_PATH = os.path.abspath(a.lib)
    _cabi.lib()
    from reversi_zero_b200.agent import model as M
    from train_bench import gpu_info
    mc = M.ModelConfig()  # ch5: 256 filters, 10 residual blocks, value_fc 256
    res = dict(gpu_info(), lib=_cabi.LIB_PATH, devices=a.devices, batch=a.batch,
               memory_taken={str(b): memory_taken(mc, a.devices, b) for b in a.max_batches},
               streams=trace(mc, a.devices, a.batch, a.steps, a.warmup))
    print(json.dumps({k: v for k, v in res.items() if k != "streams"}),
          [(len(s["kernels"]), s["memcpy"], s["memset"]) for s in res["streams"]], flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f)
