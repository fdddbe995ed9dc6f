"""Resolve time of start-sensitive and class-repeat-led general patterns: the per-unit walk (GSCAN_CHAIN=0, one GPU thread
replays the unit's loop) against the parallel path the engine picks by itself, on the same device-resident synthetic unit
(64 MiB), with identical records; then the parallel path alone on a 1 GiB unit (BIG_CASES).  Prints the GPU and its power limit beside
the numbers.

    python tools/resolve_paths_bench.py [--walk-mib 64] [--big-mib 1024] [--reps 3]   (0 MiB: leave that leg out)
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import grab_b200 as G  # noqa: E402

PATHS = {G.RESOLVE_WALK: "walk", G.RESOLVE_VM_TWO: "vm two-outcome", G.RESOLVE_VM_DENSE_TWO: "vm dense two-outcome",
         G.RESOLVE_VM_RUN_CHAIN: "class-repeat chain", G.RESOLVE_VM_ATTEMPTS: "vm attempts"}
CASES = [  # (pattern, mode, what it stands for)
    ("\\be\\w+", G.MODE_ALL, "\\b at the attempt's start (reach 1, filtered)"),
    ("(?m)^e", G.MODE_LINE, "(?m)^ (reach 1, filtered)"),
    ("(?<=[=:])\\d+", G.MODE_ALL, "one-byte look-behind (reach 1, filtered)"),
    ("\\w+@\\w+", G.MODE_ALL, "class-repeat led (run starts)"),
    ("[0-9]+\\.[0-9]+", G.MODE_LINE, "class-repeat led, LINE mode"),
    ("\\b\\w*q\\w*", G.MODE_ALL, "\\b, no candidate filter (reach 1, dense)"),
]
# the 1 GiB unit: the chain tables of a call stay within 4 GiB (<= 2 nodes per candidate), so the look-behind and the
# class-repeat cases get sparser candidates there -- with 10^8 digit or word-run candidates the engine keeps the walk
BIG_CASES = CASES[:2] + [
    ("(?<=[=:])7\\d*", G.MODE_ALL, "one-byte look-behind (reach 1, filtered)"),
    ("[xz]+\\.\\w+", G.MODE_ALL, "class-repeat led (run starts)"),
    ("[xz]+\\.\\w+", G.MODE_LINE, "class-repeat led, LINE mode"),
] + CASES[5:]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in q.split(",")]
        return name, limit
    except Exception as e:  # the numbers are still printed; say why the card is not named
        return "unknown (%s)" % e, "unknown"


def timed(ctx, pat, units, mode, reps):
    r = ctx.scan_units(pat, units, mode)  # first call sizes the buffers
    ms = []
    for _ in range(reps):
        r = ctx.scan_units(pat, units, mode)
        st = ctx.stats()
        ms.append(st["resolve_ms"])
    return r, st, float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--walk-mib", type=int, default=64)
    ap.add_argument("--big-mib", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    name, limit = gpu_info()
    print(json.dumps({"gpu": name, "power_limit": limit}))
    ctx = G.Context(0)
    ok = True
    for mib, compare in ((args.walk_mib, True), (args.big_mib, False)):
        if mib <= 0:  # 0: leave this leg out (the walk leg takes minutes)
            continue
        n = mib << 20
        d = ctx.device_alloc(n)
        try:
            ctx.synth_corpus(d, 12, 5, 1, n)  # printable ASCII, '\n' at p = 3/256 (tests/corpus.py)
            units = G.Context.device_units(d, 1, n)
            for pat_s, mode, what in (CASES if compare else BIG_CASES):
                pat = G.Pattern(pat_s)
                os.environ.pop("GSCAN_CHAIN", None)
                r_new, st_new, ms_new = timed(ctx, pat, units, mode, args.reps)
                row = {"unit_mib": mib, "pattern": pat_s, "mode": mode, "class": what, "matches": len(r_new),
                       "candidates": st_new["n_candidates"], "path": PATHS.get(st_new["resolve_path"], st_new["resolve_path"]),
                       "resolve_ms": round(ms_new, 3), "vm_limit_hit": st_new["vm_limit_hit"]}
                if compare:
                    os.environ["GSCAN_CHAIN"] = "0"
                    r_old, st_old, ms_old = timed(ctx, pat, units, mode, 1)
                    os.environ.pop("GSCAN_CHAIN", None)
                    same = len(r_old) == len(r_new) and bool(np.array_equal(r_old["start"], r_new["start"])) and \
                        bool(np.array_equal(r_old["match_len"], r_new["match_len"]))
                    ok = ok and same
                    row.update({"walk_path": PATHS.get(st_old["resolve_path"], st_old["resolve_path"]), "walk_resolve_ms": round(ms_old, 3),
                                "speedup": round(ms_old / max(ms_new, 1e-6), 1), "records_identical": same})
                print(json.dumps(row), flush=True)
        finally:
            ctx.device_free(d)
    ctx.close()
    print(json.dumps({"gpu": name, "power_limit": limit, "all_records_identical": ok}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
