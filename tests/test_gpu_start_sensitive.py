"""General patterns that look at or before an attempt's first byte (^, \\A, \\b, \\B, (?m)^, look-behinds) and patterns led by a
greedy or possessive class repeat (\\w+@\\w+) resolve in parallel on big windows: two VM attempts per candidate (the subject
beginning at the candidate, and before it) or an extra attempt where a search resumes inside a run, then the chain -- the
records stay those of the oracle's loop."""
import numpy as np
import pytest

import corpus
import grab_b200 as G
import oracle_py as O

pytestmark = pytest.mark.gpu

MiB = 1 << 20
MODES = ((G.MODE_ALL, O.MODE_ALL), (G.MODE_LINE, O.MODE_LINE), (G.MODE_FIRST, O.MODE_FIRST))

# (pattern, STRICT_REF, the resolve path it takes when the chain is forced)
FORCED = [
    ("\\bab\\b", False, G.RESOLVE_VM_TWO), ("^a\\w*", False, G.RESOLVE_VM_TWO), ("(?m)^a", False, G.RESOLVE_VM_TWO),
    ("\\Ba", False, G.RESOLVE_VM_TWO), ("(?<=a)b", False, G.RESOLVE_VM_TWO), ("(?<![ab])c\\w*", False, G.RESOLVE_VM_TWO),
    ("\\ba[ab_]*", False, G.RESOLVE_VM_TWO), ("(?<=[ =])a\\w+", False, G.RESOLVE_VM_TWO),
    ("(?<![ab])\\w+", False, G.RESOLVE_VM_DENSE_TWO), ("(?<=[ =])\\w+", False, G.RESOLVE_VM_DENSE_TWO),  # \w: too common to filter on
    ("a\\b", False, G.RESOLVE_VM_ATTEMPTS),  # the \b runs behind the attempt's first byte: start-free
    ("\\w+@\\w+", False, G.RESOLVE_VM_RUN_CHAIN), ("[ab]+c", False, G.RESOLVE_VM_RUN_CHAIN), ("\\w++b", False, G.RESOLVE_VM_RUN_CHAIN),
    ("[ab]+_", False, G.RESOLVE_VM_RUN_CHAIN), ("(?U)a+?b", False, G.RESOLVE_VM_RUN_CHAIN),
    ("(?U)a+b", False, G.RESOLVE_WALK),  # lazy leading repeat: its end can differ from inside a run
    ("(?<=ab)c", False, G.RESOLVE_WALK),  # reach 2
    ("\\b(?:a|(b))a", True, G.RESOLVE_VM_TWO), ("^(a)?b", True, G.RESOLVE_VM_TWO), ("(?<=a)(b)|c", True, G.RESOLVE_VM_TWO),
    # dense: no candidate filter
    ("\\b\\w*b_", False, G.RESOLVE_VM_DENSE_TWO), ("\\b.*c", False, G.RESOLVE_VM_DENSE_TWO), ("(?<=a)\\w*_", False, G.RESOLVE_VM_DENSE_TWO),
    ("\\b\\w*(_)a|\\b.*b_", True, G.RESOLVE_VM_DENSE_TWO),
]


def records(r, fid):
    lo, hi = np.searchsorted(r["file_id"], fid, "left"), np.searchsorted(r["file_id"], fid, "right")
    return [(int(s), int(l)) for s, l in zip(r["start"][lo:hi], r["match_len"][lo:hi])]


def test_forced_on_small_ragged_inputs(monkeypatch):
    """GSCAN_CHAIN=1 on small files: every mode, STRICT_REF on and off, lines far longer than 511 bytes (LINE mode resumes
    inside runs and right behind '\\n')."""
    monkeypatch.setenv("GSCAN_CHAIN", "1")
    rng = np.random.default_rng(11)
    bufs = [bytes(rng.choice(np.frombuffer(b"ab\n", dtype=np.uint8), size=int(n)).tobytes()) for n in [1, 2, 3, 5, 64, 511, 512, 513, 4096, 70000]]
    bufs += [bytes(rng.choice(np.frombuffer(al, dtype=np.uint8), size=n).tobytes()) for al, n in
             ((b"ab", 3000), (b"ab_ c", 5000), (b"a@b_ =c", 9000), (b"aab_ ", 9000))]
    bufs += [bufs[-1][:2000] + b"\n" + bufs[-2][:700] + b"\n" + bufs[-3][:1500]]
    bufs += [corpus.synth_file(61, i, 30000 + 977 * i).tobytes() for i in range(3)]
    ctx = G.Context(0)
    try:
        for pat, strict, path in FORCED:
            p = G.Pattern(pat, strict_ref=strict)
            o = O.Regex(pat)
            for mode, om in MODES:
                r = ctx.scan(p, bufs, mode=mode)
                st = ctx.stats()
                assert not st["vm_limit_hit"], (pat, mode)
                assert st["resolve_path"] == path, (pat, mode, st["resolve_path"])
                for i, b in enumerate(bufs):
                    assert records(r, i) == o.scan_window(b, mode=om, strict_q2=strict), (pat, mode, i, len(b))
    finally:
        ctx.close()


@pytest.mark.parametrize("pat,mode,om,path", [
    ("\\be\\w+", G.MODE_ALL, O.MODE_ALL, G.RESOLVE_VM_TWO),
    ("(?m)^e", G.MODE_LINE, O.MODE_LINE, G.RESOLVE_VM_TWO),
    ("(?<=[=:])\\d+", G.MODE_ALL, O.MODE_ALL, G.RESOLVE_VM_TWO),
    ("\\w+@\\w+", G.MODE_ALL, O.MODE_ALL, G.RESOLVE_VM_RUN_CHAIN),
    ("[0-9]+\\.[0-9]+", G.MODE_LINE, O.MODE_LINE, G.RESOLVE_VM_RUN_CHAIN),
])
def test_one_64mib_device_unit(pat, mode, om, path):
    """One 64 MiB window in device memory picks the parallel path by itself."""
    n = 64 * MiB
    host = corpus.synth_file(12, 5, n)
    ctx = G.Context(0)
    d = ctx.device_alloc(n)
    try:
        ctx.h2d(d, host)
        units = G.Context.device_units(d, 1, n)
        want = O.Regex(pat).scan_window_np(host, mode=om, strict_q2=False)
        r = ctx.scan_units(G.Pattern(pat), units, mode)
        st = ctx.stats()
        print("one 64 MiB unit, %s mode %d: %d candidates, %d matches, resolve %.3f ms, path %d"
              % (pat, mode, st["n_candidates"], len(r), st["resolve_ms"], st["resolve_path"]))
        assert st["resolve_path"] == path and not st["vm_limit_hit"]
        assert len(r) == len(want) > 1000
        assert np.array_equal(r["start"], want["start"]) and np.array_equal(r["match_len"], want["len"])
    finally:
        ctx.device_free(d)
        ctx.close()


@pytest.mark.parametrize("pat,mode,om,path", [
    ("\\be\\w+", G.MODE_LINE, O.MODE_LINE, G.RESOLVE_VM_TWO),
    ("\\w+@\\w+", G.MODE_LINE, O.MODE_LINE, G.RESOLVE_VM_RUN_CHAIN),
    ("\\b\\w*q\\w*", G.MODE_ALL, O.MODE_ALL, G.RESOLVE_VM_DENSE_TWO),
    ("\\b\\w*q\\w*", G.MODE_FIRST, O.MODE_FIRST, G.RESOLVE_VM_DENSE_TWO),
])
def test_batch_of_1mib_files(pat, mode, om, path):
    """16 files of 1 MiB pick the parallel path by themselves."""
    bufs = [corpus.synth_file(23, i, MiB) for i in range(16)]
    ctx = G.Context(0)
    try:
        r = ctx.scan(G.Pattern(pat), bufs, mode=mode)
        st = ctx.stats()
        print("16 x 1 MiB, %s mode %d: %d candidates, %d matches, resolve %.3f ms, path %d"
              % (pat, mode, st["n_candidates"], len(r), st["resolve_ms"], st["resolve_path"]))
        assert st["resolve_path"] == path and not st["vm_limit_hit"]
        o = O.Regex(pat)
        total = 0
        for i, b in enumerate(bufs):
            want = o.scan_window(b.tobytes(), mode=om, strict_q2=False)
            assert records(r, i) == want, (pat, mode, i)
            total += len(want)
        assert total > (10 if mode == G.MODE_FIRST else 1000)
    finally:
        ctx.close()
