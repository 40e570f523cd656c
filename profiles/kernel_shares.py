#!/usr/bin/env python
"""Which kernels the GPU time of bench.py's `value` regime goes to: sm_align_pairs with 16 pipelines on
their own streams, 2 host threads, device-resident pairs (bench.PairData), knn_queries_per_cta 1024, 30
fixed iterations, batches of 64 alignments.  After a warm-up the steps run under torch.profiler with CUDA
activities; the device time of every kernel (and copy / memset) is summed per name and printed with its
share of the total, next to the card's name and power limit.  Kernels of different alignments overlap,
so the shares are of summed kernel time, not of wall time.

    python profiles/kernel_shares.py [--steps 5] [--warmup 2] [--out DIR]
"""
import argparse
import collections
import json
import os
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
import torch  # noqa: E402
from torch.autograd import DeviceType  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402
import bench  # noqa: E402
import staticmapping_b200 as smb  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "kernel_shares"),
                    help="directory of the trace and the JSON (default: a directory under the system's temporary one)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kernel_shares.py needs a CUDA device")
    steps = max(5, args.steps)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    P, T, B = 16, 2, 64
    data = [bench.PairData(smb, torch, dev, 0, w) for w in range(P)]
    matchers, streams = [], []
    for _ in range(P):
        m = smb.IcpFast(0)
        m.InitWithXml({"max_iteration": bench.ITERATIONS, "disable_convergence_check": 1, "knn_queries_per_cta": 1024})
        s = torch.cuda.Stream(device=dev)
        m.SetStream(s.cuda_stream)
        matchers.append(m); streams.append(s)
    pairs = [data[k % P].pair(False) for k in range(B)]

    def run(n):
        def body(j):
            for _ in range(n):
                smb.AlignPairs(matchers[j::T], pairs[j::T])
        ths = [threading.Thread(target=body, args=(j,)) for j in range(T)]
        torch.cuda.synchronize(); t0 = time.perf_counter()
        for t in ths: t.start()
        for t in ths: t.join()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    run(args.warmup)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        secs = run(steps)
    os.makedirs(args.out, exist_ok=True)
    prof.export_chrome_trace(os.path.join(args.out, "kernel_shares.pt.trace.json"))

    total_us, count = collections.Counter(), collections.Counter()
    for e in prof.events():
        if e.device_type == DeviceType.CUDA:
            total_us[e.name] += e.time_range.elapsed_us()
            count[e.name] += 1
    whole = sum(total_us.values())
    gpu = bench.gpu_identity(0, torch.cuda.get_device_name(dev))
    n_align = steps * B
    print(f"card: {gpu['name']}, power limit {gpu['power_limit_w']} W")
    print(f"{n_align} alignments in {secs * 1e3:.1f} ms under the profiler ({n_align / secs:.1f} alignments/s, "
          f"profiler on); summed device time {whole / 1e3:.1f} ms")
    print(f"{'share':>7} {'ms':>9} {'us/alignment':>13} {'launches':>9}  name")
    rows = []
    for name, us in total_us.most_common():
        rows.append({"name": name, "ms": us / 1e3, "share": us / whole, "launches": count[name],
                     "us_per_alignment": us / n_align})
        print(f"{100 * us / whole:6.2f}% {us / 1e3:9.2f} {us / n_align:13.2f} {count[name]:9d}  {name[:120]}")
    with open(os.path.join(args.out, "kernel_shares.json"), "w") as f:
        json.dump({"gpu": gpu, "alignments": n_align, "seconds_profiled": secs, "kernels": rows}, f, indent=1)
    print(f"trace and JSON in {args.out}")
    torch.cuda.synchronize()
    for m in matchers:
        m.SetStream(0)
        m.__del__()


if __name__ == "__main__":
    main()
