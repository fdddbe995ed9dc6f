"""The segment occupancy bits of one context across scans: the scan kernels set one bit per non-empty segment and the
resolve reads only those entries and clears the bits it read.  An overflow re-scan (the candidate buffer grows and the
batch is scanned again under the same generation tag), a sparse scan behind it, and a smaller batch behind that must
all give the records of a fresh context and of the oracle."""
import numpy as np
import pytest

import corpus
import grab_b200 as G
import oracle_py as O

pytestmark = pytest.mark.gpu

N_FILES, FILE_LEN, SEED, NEEDLE, EVERY = 256, 1 << 20, 3, b"foobardoesexist", 64


def by_file(r):
    out = {}
    for f, s, l in zip(r["file_id"].tolist(), r["start"].tolist(), r["match_len"].tolist()):
        out.setdefault(f, []).append((s, l))
    return out


def test_overflow_rescan_then_sparse_scans_on_one_context():
    ctx, fresh = G.Context(0), None
    d = ctx.device_alloc(N_FILES * FILE_LEN)
    try:
        ctx.synth_corpus(d, SEED, 0, N_FILES, FILE_LEN, needle=NEEDLE, needle_every=EVERY)
        batch = ctx.batch_create(G.Context.device_units(d, N_FILES, FILE_LEN))
        # one byte of the synthetic text: ~3 M candidates over 256 MiB, more than the 1 Mi slots a new context starts with
        dense = ctx.batch_scan(G.Pattern("e", literal=True), batch)
        st = ctx.stats()
        assert st["scan_launches"] == 2 and st["n_candidates"] > (1 << 20), st
        got = by_file(dense)
        o = O.Regex("e", literal=True)
        for f in list(range(0, N_FILES, 16)) + [N_FILES - 1]:
            want = o.scan_window(corpus.synth_file(SEED, f, FILE_LEN, NEEDLE, EVERY).tobytes())
            assert got.get(f, []) == want, f

        # behind it on the same context: the sparse headline pattern, then a batch of fewer segments
        sparse = ctx.batch_scan(G.Pattern(NEEDLE.decode(), literal=True), batch)
        assert ctx.stats()["scan_launches"] == 1
        planted = [f for f in range(N_FILES) if f % EVERY == EVERY // 2]
        assert sorted(by_file(sparse)) == planted
        for f in planted:
            assert by_file(sparse)[f] == [(corpus.needle_offset(SEED, f, FILE_LEN, len(NEEDLE)), len(NEEDLE))]
        small = ctx.batch_create(G.Context.device_units(d + 30 * FILE_LEN, 8, FILE_LEN, first_file_id=30))
        few = ctx.batch_scan(G.Pattern("foo", literal=True), small)

        fresh = G.Context(0)
        assert fresh.batch_scan(G.Pattern("e", literal=True), batch).tobytes() == dense.tobytes()
        fresh2 = G.Context(0)
        assert fresh2.batch_scan(G.Pattern(NEEDLE.decode(), literal=True), batch).tobytes() == sparse.tobytes()
        fresh2.close()
        assert fresh.batch_scan(G.Pattern("foo", literal=True), small).tobytes() == few.tobytes()
        o = O.Regex("foo", literal=True)
        for f in range(30, 38):
            want = o.scan_window(corpus.synth_file(SEED, f, FILE_LEN, NEEDLE, EVERY).tobytes())
            assert by_file(few).get(f, []) == want, f
        small.free()
        batch.free()
    finally:
        if fresh is not None:
            fresh.close()
        ctx.device_free(d)
        ctx.close()
