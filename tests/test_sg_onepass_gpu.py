"""ma_sg_gen emits each read's sorted arcs and both index words in one pass over the hits (tiles of reads with a look-back for
their offsets).  It must give what the oracle port gives: the arcs, idx and seq after ma_sg_gen, and the arcs and idx after
asg_arc_del_trans.  The hit sets are made by hand so that they
reach every case: read counts around the tile size, reads without arcs, reads on both sides of 256 and 8192 hits (beyond 8192
the whole graph takes the column sort), reads deleted by a contained hit and by the palindromic self-hit, unsorted query ids
and no hits at all.  In the fused path the per-read bounds come from the read selection: the raw graph after mab_select is
compared step by step, and it must be built without a device-wide sort.  The fused paths (hits from mab_load_hits, the sharded
layout with one rank and with the all-gather branch) are held to the port's GFA."""
import ctypes as C

import numpy as np
import pytest

from miniasm_b200 import capi, synth
from miniasm_b200.capi import HIT_DT, SUB_DT
from miniasm_b200.pipeline import Pipeline, canon_arcs

pytestmark = pytest.mark.gpu

L, S = 10000, 1500   # read length, distance between the starts of consecutive reads


def make_hits(n_reads, hub_sizes=(), seed=1, contained=(), palindromes=(), internal_only=()):
    """Reads 0 ..< n_reads of length L, each overlapping a few later reads at both ends (arcs of both directions); hub k (ids
    after the plain reads) has hub_sizes[k] dovetail hits.  contained: reads that also hold a hit contained in a longer target;
    palindromes: reads with a reverse self-hit on the diagonal; internal_only: reads whose only hits are internal matches."""
    rng = np.random.default_rng(seed)
    n_hub = len(hub_sizes)
    n_seq = n_reads + n_hub + 1                       # the last read is the long target of the contained hits
    big = n_seq - 1
    lens = np.full(n_seq, L, dtype=np.uint32)
    lens[big] = L + 400
    rows = []

    def hit(q, qs, qe, t, ts, te, rev=0):
        rows.append((q << 32 | qs, qe, t, ts, te, (qe - qs) // 2 | rev << 31, qe - qs))

    for q in range(n_reads):                          # read q starts at q * S of one genome: overlaps make transitive arcs
        if q in internal_only:
            hit(q, 3000, 5000, (q + 1) % n_reads, 3000, 5000)
            continue
        for t in range(q + 1, min(q + 6, n_reads)):
            if t in internal_only or rng.random() < .2:
                continue
            ov = L - (t - q) * S
            hit(q, L - ov, L, t, 0, ov)               # q's 3' end onto t's 5' end: an arc leaving q+
            hit(t, 0, ov, q, L - ov, L)               # and the same overlap seen from t: an arc leaving t-
        if q in contained:
            hit(q, 0, L, big, 200, 200 + L)
        if q in palindromes:
            hit(q, 3000, L, q, 3000, L, rev=1)
    for k, m in enumerate(hub_sizes):
        q = n_reads + k
        for j in range(m):
            ov = 2000 + (j * 7919) % 7000
            t = j % n_reads
            if j % 3:
                hit(q, L - ov, L, t, 0, ov, rev=j & 1)
            else:
                hit(q, 0, ov, t, L - ov, L)
    a = np.array(rows, dtype=np.uint64).reshape(-1, 7) if rows else np.zeros((0, 7), dtype=np.uint64)
    h = np.zeros(len(a), dtype=HIT_DT)
    for i, f in enumerate(["qns", "qe", "tn", "ts", "te", "ml_rev", "bl_del"]):
        h[f] = a[:, i]
    h = h[np.argsort(h["qns"], kind="stable")]
    return h, lens


def graph_states(lib, hits, lens):
    """(graph after ma_sg_gen, graph after asg_arc_del_trans) from the given hits, with every read kept whole."""
    p = Pipeline(lib, b"")
    p.d = lib.sd_init()
    for i, ln in enumerate(lens):
        lib.sd_put(p.d, f"r{i}".encode(), int(ln))
    p.hits, p.n_hits = capi.c_malloc_copy(hits), len(hits)
    sub = np.zeros(len(lens), dtype=SUB_DT)
    sub["e"] = lens
    p.sub = capi.c_malloc_copy(sub)
    p.sg_gen()

    def state():
        a, s, i, srt, _ = p.graph_np()
        return [srt, s.copy(), None if i is None else i.copy(), a["ul"].copy(), canon_arcs(a)]

    out = [state()]
    p.clean(upto=6)
    out.append(state())
    p.free()
    return out


def check_same(got, want):
    for g, w in zip(got, want):
        assert g[0] == w[0]
        for x, y in zip(g[1:], w[1:]):
            assert (x is None) == (y is None)
            if x is not None:
                assert len(x) == len(y) and np.array_equal(x, y)


CASES = {
    "one_tile_short": dict(n_reads=5),
    "tiles_plus_rest": dict(n_reads=8 * 37 + 5),
    "many_tiles": dict(n_reads=20000, internal_only=tuple(range(0, 20000, 97))),
    "warp_and_cta_reads": dict(n_reads=400, hub_sizes=(255, 256, 257, 1000, 8192)),
    "column_sort_read": dict(n_reads=400, hub_sizes=(100, 8193)),
    "deleted_reads": dict(n_reads=600, contained=(3, 50, 51, 599), palindromes=(7, 8, 300)),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_sg_gen_and_del_trans(case, port, prod):
    hits, lens = make_hits(**CASES[case])
    got, want = graph_states(prod, hits, lens), graph_states(port, hits, lens)
    check_same(got, want)
    if case == "deleted_reads":
        assert (want[0][1] >> 31).sum() > 0           # reads were deleted, so asg_arc_rm had arcs to remove
    assert len(want[0][3]) > len(want[1][3]) > 0      # the reduction removed arcs and kept some


def test_unsorted_query_ids(port, prod):
    hits, lens = make_hits(n_reads=300, hub_sizes=(300,), contained=(5,))
    hits = hits[np.random.default_rng(2).permutation(len(hits))]
    check_same(graph_states(prod, hits, lens), graph_states(port, hits, lens))


def test_no_hits(port, prod):
    hits, lens = make_hits(n_reads=20)
    check_same(graph_states(prod, hits[:0], lens), graph_states(port, hits[:0], lens))


def fused_gfa(prod, port, paf, how):
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    if how == "hits":
        p = Pipeline(port, paf).read()
        assert prod.mab_load_hits(ctx, p.hits, p.n_hits, p.d) == 0
        p.free()
        prod.mab_select(ctx, C.byref(opt), 0, 0, 100)
        prod.mab_layout(ctx, C.byref(opt), 100)
    else:
        data = open(paf, "rb").read()
        assert prod.mab_load_paf_text(ctx, data, len(data)) == 0
        assert prod.mab_shard_init(ctx, 0, 1, None) == 0
        prod.mab_ingest_sharded(ctx, opt.min_span, opt.min_match, 1)
        prod.mab_select_sharded(ctx, C.byref(opt))
        prod.mab_layout_sharded(ctx, C.byref(opt))
    prod.mab_unitigs(ctx)
    d, sub, ug = prod.mab_export_dict(ctx), prod.mab_export_sub(ctx), prod.mab_export_ug(ctx)
    gfa = prod.print_to_string("ma_ug_print", ug, d, sub)
    prod.ma_ug_destroy(ug), capi.c_free(sub), prod.sd_destroy(d), prod.mab_destroy(ctx)
    return gfa


@pytest.mark.parametrize("how", ["hits", "sharded_p2p", "sharded_allgather"])
@pytest.mark.parametrize("name", ["chaos_small", "bubbles800"])
def test_fused_layout(name, how, paf_dir, port, prod, monkeypatch):
    paf = synth.generate(name, f"{paf_dir}/onepass_{name}.paf")
    monkeypatch.setenv("MAB_SHARD_P2P", "0" if how == "sharded_allgather" else "1")
    want = Pipeline(port, paf).run_all()
    assert fused_gfa(prod, port, paf, "hits" if how == "hits" else "sharded") == want


@pytest.mark.parametrize("name", ["chaos_small", "bubbles800", "skew_small"])
def test_fused_raw_graph_after_selection(name, paf_dir, port, prod):
    """mab_layout at stage 5 builds the raw graph from the bounds the selection handed over: same graph as the port's
    ma_sg_gen after its selection, and no library call (the column sort is a CUB radix sort) on the way."""
    paf = synth.generate(name, f"{paf_dir}/onepass_{name}.paf")
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    data = open(paf, "rb").read()
    assert prod.mab_load_paf_text(ctx, data, len(data)) == 0
    prod.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    prod.mab_select(ctx, C.byref(opt), 0, 0, 100)
    n_lib = prod.mab_stats(ctx).contents.n_lib_calls
    prod.mab_layout(ctx, C.byref(opt), 5)
    lib_calls = prod.mab_stats(ctx).contents.n_lib_calls - n_lib
    g = prod.mab_export_sg(ctx)
    a, s, i, srt, _ = prod.read_graph(g)
    got = [srt, s.copy(), i.copy(), a["ul"].copy(), canon_arcs(a)]
    if not (s >> 31).any():                           # with a deleted read, asg_arc_rm's compaction is a library call too
        assert lib_calls == 0
    prod.asg_destroy(g), prod.mab_destroy(ctx)
    r = Pipeline(port, paf).read().select().sg_gen()
    a, s, i, srt, _ = r.graph_np()
    want = [srt, s.copy(), i.copy(), a["ul"].copy(), canon_arcs(a)]
    r.free()
    check_same([got], [want])
