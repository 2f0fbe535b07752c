"""The default read selection leaves the kept hits in their reads' buckets, under the old read ids (DHits::map), and ma_sg_gen
reads them there: it renumbers each hit in registers and skips a hit whose target was dropped before classifying it, so that
the dropped hit's deletion side effects (a contained query, the palindromic self-hit) do not happen.  Every other reader of
the hits first writes the dense array.  Held to the oracle port on a hand-made file: reads removed by containment that kept
reads still hold hits to, one such hit that the layout's options classify as a contained query, palindromic self-hits, hub
reads whose buckets hold 257..8192 hits (and, in two more files, beyond 8192) with kept counts on both sides of 256, and reads left without
hits.  The layout runs twice on one selection; the hits and the -p paf text are read after a layout has read the buckets;
the sharded path with one rank goes the same way.  ma_hit_sub's per-read key sort is held to the port through the drop-in on
hand-made reads: start keys in order or not, duplicates, and key counts on both sides of every width of the register network."""
import ctypes as C

import numpy as np
import pytest

from miniasm_b200 import capi
from miniasm_b200.capi import HIT_DT, SUB_DT
from miniasm_b200.pipeline import Pipeline, canon_arcs
from tests.test_dump_writers_cpu import py_paf

pytestmark = pytest.mark.gpu

L, S = 10000, 1500           # chain reads: length, distance between the starts of consecutive reads
N_CHAIN = 120
CONTAINED = (20, 40, 41, 90)  # chain reads that hold a short read contained in them
NEAR = (30, 60)               # chain reads with an internal match to a read the selection drops (contained in a long read)
PALINDROMES = (50, 51)
# hub reads: (hits to one kept chain read, short partner reads contained in the hub; each gives the hub three hits)
HUBS = ((250, 20), (256, 20), (260, 20), (300, 600))
# a bucket beyond 8192 hits of which 100 are kept (the CTA tier reads it), and a read that keeps more than 8192 (the column sort,
# which reads the dense array)
BIG_HUBS = {"bucket_beyond_8192": (100, 2800), "column_sort": (8200, 20)}


def write_buckets_paf(path, hubs=HUBS):
    lines = []

    def line(q, ql, qs, qe, t, tl, ts, te, strand="+"):
        lines.append(f"{q}\t{ql}\t{qs}\t{qe}\t{strand}\t{t}\t{tl}\t{ts}\t{te}\t{(qe - qs) // 2}\t{qe - qs}\t255\n")

    for i in range(N_CHAIN):
        for j in range(i + 1, min(i + 7, N_CHAIN)):
            ov = L - (j - i) * S
            line(f"a{i}", L, L - ov, L, f"a{j}", L, 0, ov)
    for k in CONTAINED:           # c{k} lies inside a{k-2} .. a{k+2}: deleted as contained; those reads keep hits to it
        for j in range(k - 2, k + 3):
            x = (k - j) * S + 3000
            line(f"c{k}", 4000, 0, 4000, f"a{j}", L, x, x + 4000)
    for k in NEAR:                # a{k} -> b{k}: internal at the selection's max_hang (1000), a contained query at 2000;
        line(f"a{k}", L, 1500, L, f"b{k}", 12000, 2000, 10500)    # b{k} is contained in u{k}, and u{k} keeps no hit
        for _ in range(3):
            line(f"b{k}", 12000, 0, 12000, f"u{k}", 20000, 4000, 16000)
            line(f"w{k}", 6000, 0, 6000, f"u{k}", 20000, 0, 6000)
    for k in PALINDROMES:
        line(f"a{k}", L, 3000, L, f"a{k}", L, 3000, L, "-")
    for h, (n_kept, n_part) in enumerate(hubs):
        anchor = 10 + 15 * h
        for _ in range(n_kept):
            line(f"h{h}", 20000, 14000, 20000, f"a{anchor}", L, 0, 6000)
        for j in range(n_part):
            x = (j * 7919) % 14000
            for _ in range(3):
                line(f"p{h}_{j}", 6000, 0, 6000, f"h{h}", 20000, x, x + 6000)
    with open(path, "w") as f:
        f.writelines(lines)
    return path


@pytest.fixture(scope="module")
def paf(paf_dir):
    return write_buckets_paf(f"{paf_dir}/buckets.paf")


@pytest.fixture(scope="module")
def paf_big(paf_dir):
    return {k: write_buckets_paf(f"{paf_dir}/buckets_{k}.paf", HUBS + (v,)) for k, v in BIG_HUBS.items()}


def layout_opt(lib, wide):
    o = lib.default_opt()
    if wide:
        o.max_hang = 2000
    return o


def is_qcont(h, ql, tl, o):
    """mab_hit2arc's contained-query verdict (hit2arc.cuh), for the small positive values of the hand-made file"""
    qs, qe, ts, te = int(h["qns"]) & 0xffffffff, int(h["qe"]), int(h["ts"]), int(h["te"])
    tl5, tl3 = (tl - te, ts) if int(h["ml_rev"]) >> 31 else (ts, tl - te)
    q3 = ql - qe
    ext5, ext3 = min(qs, tl5), min(q3, tl3)
    span, full = qe - qs, qe - qs + min(qs, tl5) + min(q3, tl3)
    if ext5 > o.max_hang or ext3 > o.max_hang or np.float32(span) < np.float32(full) * np.float32(o.int_frac):
        return False
    return qs <= tl5 and q3 <= tl3


def test_buckets_paf_reaches_every_case(paf, port):
    """Kept reads hold hits to dropped reads, one of them a contained query under the wide layout options; hub buckets hold
    257..8192 hits, with kept counts on both sides of 256; some kept reads are left without hits; a palindromic self-hit
    survives."""
    p = Pipeline(port, paf).read().sub1().cut().flt().sub2_cut_merge()
    names = p.names()
    hits, sub = p.hits_np().copy(), p.sub_np().copy()
    p.contained()
    kept = set(p.names())
    kept_hits = p.hits_np()
    p.free()
    q = (hits["qns"] >> np.uint64(32)).astype(np.int64)
    t = hits["tn"].astype(np.int64)
    is_kept = np.array([n in kept for n in names])
    live_q = is_kept[q]
    dropped_t = live_q & ~is_kept[t]
    assert dropped_t.sum() > 0
    lens = (sub["e"] - (sub["s_del"] & 0x7fffffff)).astype(np.int64)
    wide = layout_opt(port, True)
    assert any(is_qcont(hits[i], lens[q[i]], lens[t[i]], wide) for i in np.flatnonzero(dropped_t))
    bucket = np.bincount(q[live_q], minlength=len(names))
    surv = np.bincount((kept_hits["qns"] >> np.uint64(32)).astype(np.int64), minlength=len(kept))
    hub_ids = [names.index(f"h{h}".encode()) for h in range(len(HUBS))]
    assert [int(bucket[i]) for i in hub_ids] == [n + 3 * m for n, m in HUBS]
    kept_names = [n for n in names if n in kept]
    assert sorted(int(surv[kept_names.index(f"h{h}".encode())]) for h in range(len(HUBS))) == sorted(n for n, _ in HUBS)
    assert (surv == 0).any()
    kq = (kept_hits["qns"] >> np.uint64(32))
    assert (kq == kept_hits["tn"]).any()


def graph_of(lib, g):
    a, s, i, srt, _ = lib.read_graph(g)
    return [srt, s.copy(), None if i is None else i.copy(), a["ul"].copy(), canon_arcs(a)]


def port_raw_graph(port, paf, wide):
    p = Pipeline(port, paf).read().select()
    p.opt = layout_opt(port, wide)
    p.sg_gen()
    a, s, i, srt, _ = p.graph_np()
    out = [srt, s.copy(), None if i is None else i.copy(), a["ul"].copy(), canon_arcs(a)]
    names = p.names()
    p.free()
    return out, names


def check_same(got, want):
    assert got[0] == want[0]
    for x, y in zip(got[1:], want[1:]):
        assert (x is None) == (y is None)
        if x is not None:
            assert len(x) == len(y) and np.array_equal(x, y)


def selected_ctx(prod, paf, sharded=False):
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    data = open(paf, "rb").read()
    assert prod.mab_load_paf_text(ctx, data, len(data)) == 0
    if sharded:
        assert prod.mab_shard_init(ctx, 0, 1, None) == 0
        prod.mab_ingest_sharded(ctx, opt.min_span, opt.min_match, 1)
        prod.mab_select_sharded(ctx, C.byref(opt))
    else:
        prod.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
        prod.mab_select(ctx, C.byref(opt), 0, 0, 100)
    return ctx


@pytest.mark.parametrize("big", [None] + sorted(BIG_HUBS))
@pytest.mark.parametrize("wide", [False, True], ids=["default_opt", "wide_hang"])
def test_raw_graph_twice(paf, paf_big, port, prod, wide, big):
    """mab_layout at stage 5 twice on one selection, with the layout's own options: both graphs are the port's."""
    paf = paf_big[big] if big else paf
    want, names = port_raw_graph(port, paf, wide)
    deleted = {n for n, s in zip(names, want[1]) if s >> 31}
    assert {f"a{k}".encode() for k in PALINDROMES} <= deleted
    assert not {f"a{k}".encode() for k in NEAR} & deleted   # their contained-query hits go to dropped reads
    ctx = selected_ctx(prod, paf)
    o = layout_opt(prod, wide)
    for _ in range(2):
        prod.mab_layout(ctx, C.byref(o), 5)
        g = prod.mab_export_sg(ctx)
        check_same(graph_of(prod, g), want)
        prod.asg_destroy(g)
    prod.mab_destroy(ctx)


def port_selection(port, paf):
    p = Pipeline(port, paf).read().select()
    out = {"hits": p.hits_np().copy(), "sub": p.sub_np().copy(), "names": p.names()}
    gfa = Pipeline(port, paf).run_all()
    p.free()
    return out, gfa


def masked(h):
    h = h.copy()
    h["bl_del"] &= 0x7fffffff
    return h


def gfa_of(prod, ctx):
    d, sub, ug = prod.mab_export_dict(ctx), prod.mab_export_sub(ctx), prod.mab_export_ug(ctx)
    gfa = prod.print_to_string("ma_ug_print", ug, d, sub)
    prod.ma_ug_destroy(ug), capi.c_free(sub), prod.sd_destroy(d)
    return gfa


@pytest.mark.parametrize("first", ["export_hits", "write_paf"])
def test_hits_after_layout(paf, port, prod, first, tmp_path):
    """After a full layout has read the buckets (and a second one at stage 5), the GFA, the exported hits and the -p paf text
    are the port's, whichever reader writes the dense array."""
    want, want_gfa = port_selection(port, paf)
    want_paf = py_paf(masked(want["hits"]), want["names"], want["sub"])
    ctx = selected_ctx(prod, paf)
    opt = prod.default_opt()
    prod.mab_layout(ctx, C.byref(opt), 100)
    prod.mab_unitigs(ctx)
    assert gfa_of(prod, ctx) == want_gfa
    prod.mab_layout(ctx, C.byref(opt), 5)

    def paf_text():
        path = str(tmp_path / "o.paf")
        fp = capi._libc.fopen(path.encode(), b"w")
        n = prod.mab_write_paf(ctx, fp)
        capi._libc.fclose(fp)
        text = open(path, "rb").read()
        assert n == len(text)
        return text

    def hits():
        n = C.c_size_t(0)
        hp = prod.mab_export_hits(ctx, C.byref(n))
        h = masked(capi.np_from_ptr(hp, n.value, HIT_DT))
        capi.c_free(hp)
        return h

    if first == "write_paf":
        assert paf_text() == want_paf
    got = hits()
    assert len(got) == len(want["hits"]) and np.array_equal(got, masked(want["hits"]))
    assert paf_text() == want_paf
    assert prod.mab_stats(ctx).contents.n_hits_final == len(want["hits"])
    prod.mab_layout(ctx, C.byref(opt), 100)           # the dense array from here on
    prod.mab_unitigs(ctx)
    assert gfa_of(prod, ctx) == want_gfa
    prod.mab_destroy(ctx)


def test_select_again_after_layout(paf, port, prod):
    """A second selection on a selected context starts from the dense array: the port's two selections in turn."""
    p = Pipeline(port, paf).read().select().select()
    want = masked(p.hits_np())
    p.free()
    ctx = selected_ctx(prod, paf)
    opt = prod.default_opt()
    prod.mab_layout(ctx, C.byref(opt), 5)
    prod.mab_select(ctx, C.byref(opt), 0, 0, 100)
    n = C.c_size_t(0)
    hp = prod.mab_export_hits(ctx, C.byref(n))
    got = masked(capi.np_from_ptr(hp, n.value, HIT_DT))
    capi.c_free(hp), prod.mab_destroy(ctx)
    assert len(got) == len(want) and np.array_equal(got, want)


def sub_case_hits(n_keys, order, seed=3):
    """One read (id 0) with n_keys hits that emit sub keys, plus a self-hit and a low-identity hit that emit none.  order:
    "sorted" (qs order, as the bucket sort leaves it), "shuffled", "wrap" (one start at qs + clip >= 2^31, where the key
    wraps) or "ties" (duplicate starts, and a start at the coordinate of another hit's end)."""
    rng = np.random.default_rng(seed + n_keys)
    qs = np.sort(rng.integers(0, 30000, n_keys)).astype(np.uint64)
    qe = qs + rng.integers(3000, 9000, n_keys).astype(np.uint64)
    if order == "ties":
        qs[1::3] = qs[0:-1:3][: len(qs[1::3])]
        qs[-1] = qe[0] - 2000                      # start + clip == the first hit's end - clip at clip 1000
        qe[-1] = max(int(qe[-1]), int(qs[-1]) + 3000)
        idx = np.argsort(qs, kind="stable")
        qs, qe = qs[idx], qe[idx]
    if order == "wrap":
        qs[-1], qe[-1] = (1 << 31) - 500, (1 << 31) + 6000
    h = np.zeros(n_keys + 2, dtype=HIT_DT)
    h["qns"][:n_keys], h["qe"][:n_keys] = qs, qe
    h["tn"][:n_keys] = 1 + np.arange(n_keys) % 7
    h["ml_rev"][:n_keys], h["bl_del"][:n_keys] = (qe - qs) // 2, qe - qs
    h[n_keys] = (100, 8000, 0, 100, 8000, 4000, 7900)        # self-hit
    h[n_keys + 1] = (200, 9000, 2, 0, 8800, 1, 8800)         # identity below min_iden
    if order == "shuffled":
        h = h[rng.permutation(len(h))]
    return h


@pytest.mark.parametrize("clip", [0, 1000])
@pytest.mark.parametrize("order", ["sorted", "shuffled", "wrap", "ties"])
@pytest.mark.parametrize("n_keys", [1, 31, 32, 33, 64, 65, 128, 129, 200, 256])
def test_sub_key_runs(n_keys, order, clip, port, prod):
    """ma_hit_sub through the drop-in: start keys in order or not (shuffled hits, a key that wraps past 2^32), duplicate starts,
    a start on an end, key counts on both sides of every network width"""
    h = sub_case_hits(n_keys, order)
    o = prod.default_opt()
    subs = []
    for lib in (prod, port):
        p = capi.c_malloc_copy(h)
        s = lib.ma_hit_sub(o.min_dp, o.min_iden, clip, len(h), p, 8)
        subs.append(capi.np_from_ptr(s, 8, SUB_DT).copy())
        capi.c_free(s), capi.c_free(p)
    assert np.array_equal(subs[0], subs[1])


def test_sharded_one_rank(paf, port, prod):
    want = Pipeline(port, paf).run_all()
    ctx = selected_ctx(prod, paf, sharded=True)
    opt = prod.default_opt()
    prod.mab_layout_sharded(ctx, C.byref(opt))
    prod.mab_unitigs(ctx)
    assert gfa_of(prod, ctx) == want
    prod.mab_destroy(ctx)
