#!/usr/bin/env python
"""Where the time of the headline step goes (BASELINE configs[1]: literal 'foobardoesexist', 32 GiB of 1 MiB files,
seed 2, needle every 64 files, ALL mode), for whichever library GSCAN_LIB names.

After warm-up it prints, as the median and min-max over --calls calls:
  read_probe_gbs   k_read_probe over the corpus (what the card's LSU path reads)
  null_ring_gbs    gscan_tma_probe geom 0: the stream geometry's TMA ring with a consumer that looks at nothing
  kernel_gbs       the headline scan kernel
  resolve_ms       the resolve kernels of the call (CUDA events)
  host_in_call_ms  total_ms - scan kernel - resolve: host time inside gscan_batch_scan
  caller_ms        wall time between the starts of consecutive calls - total_ms: time outside the call

--trace DIR instead records five headline steps with torch.profiler (CUDA activities) to DIR/step_budget.pt.trace.json
and prints the kernels of one step with the GPU-idle gap in front of each.

Usage: [GSCAN_LIB=...] python tools/step_budget.py [--gib 32] [--calls 12] [--trace DIR]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PATTERN, SEED, NEEDLE_EVERY, FILE_LEN = "foobardoesexist", 2, 64, 1 << 20


def spread(v):
    v = sorted(v)
    return {"median": v[len(v) // 2], "min": v[0], "max": v[-1]}


def trace(ctx, pat, batch, G, out_dir):
    from torch.profiler import profile, ProfilerActivity
    for _ in range(3):
        ctx.batch_scan(pat, batch, G.MODE_ALL, copy=False)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            ctx.batch_scan(pat, batch, G.MODE_ALL, copy=False)
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "step_budget.pt.trace.json")
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))["traceEvents"]
          if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    ev.sort(key=lambda e: e["ts"])
    # one step = from a scan kernel to the event before the next scan kernel; print the second-to-last full one
    starts = [i for i, e in enumerate(ev) if e["name"].startswith("void gscan::scan_kernel")]
    a, b = starts[-2], starts[-1]
    rows, idle = [], 0.0
    for i in range(a, b):
        gap = ev[i]["ts"] - (ev[i - 1]["ts"] + ev[i - 1]["dur"]) if i > a else 0.0
        idle += gap
        rows.append({"name": ev[i]["name"][:90], "dur_us": ev[i]["dur"], "gap_before_us": gap})
    step_us = ev[b]["ts"] - ev[a]["ts"]
    print(json.dumps({"trace": path, "step_us": step_us, "gpu_idle_us": idle + (ev[b]["ts"] - ev[b - 1]["ts"] - ev[b - 1]["dur"]),
                      "events": rows}, indent=1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=int, default=32)
    ap.add_argument("--calls", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--trace", metavar="DIR", default=None)
    a = ap.parse_args()

    import grab_b200 as G
    ctx = G.Context(0)
    n = a.gib * 1024
    nbytes = n * FILE_LEN
    d = ctx.device_alloc(nbytes)
    ctx.synth_corpus(d, SEED, 0, n, FILE_LEN, needle=PATTERN.encode(), needle_every=NEEDLE_EVERY)
    batch = ctx.batch_create(G.Context.device_units(d, n, FILE_LEN))
    pat = G.Pattern(PATTERN, literal=True)
    if a.trace:
        trace(ctx, pat, batch, G, a.trace)
        return

    for _ in range(a.warmup):
        ctx.batch_scan(pat, batch, G.MODE_ALL, copy=False)
        ctx.tma_probe(batch, 0)
        ctx.read_probe(d, nbytes)
    probe = [nbytes / (ctx.read_probe(d, nbytes)[0] * 1e-3) / 1e9 for _ in range(a.calls)]
    null = [nbytes / (ctx.tma_probe(batch, 0) * 1e-3) / 1e9 for _ in range(a.calls)]
    kern, res, host, caller, total, t_start = [], [], [], [], [], []
    for _ in range(a.calls + 1):
        t_start.append(time.perf_counter())
        r = ctx.batch_scan(pat, batch, G.MODE_ALL, copy=False)
        st = ctx.stats()
        kern.append(st["scan_kernel_ms"])
        res.append(st["resolve_ms"])
        total.append(st["total_ms"])
        host.append(st["total_ms"] - st["scan_kernel_ms"] - st["resolve_ms"])
    for i in range(a.calls):
        caller.append((t_start[i + 1] - t_start[i]) * 1e3 - total[i])
    out = {"lib": os.path.basename(G.LIB_PATH), "bytes": nbytes, "matches": int(len(r)),
           "read_probe_gbs": spread(probe), "null_ring_gbs": spread(null),
           "kernel_gbs": spread([nbytes / (k * 1e-3) / 1e9 for k in kern[:a.calls]]),
           "kernel_ms": spread(kern[:a.calls]), "resolve_ms": spread(res[:a.calls]), "host_in_call_ms": spread(host[:a.calls]),
           "caller_ms": spread(caller), "call_interval_ms": spread([(t_start[i + 1] - t_start[i]) * 1e3 for i in range(a.calls)])}
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
