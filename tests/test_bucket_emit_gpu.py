"""The ingest emits every hit straight into its query read's bucket, with an ordinal (2 * line, + 1 for the mirrored hit) in
place of the query id, and the bucket sort orders each bucket by (qs, ordinal).  The result must be exactly the oracle port's
stable ma_hit_sort order, element for element.  The hand-made PAF puts long runs of equal (qid, qs) together with every kind
of line that changes what a line emits: lines the store filter drops, 10-field lines (bl carried from an earlier line), self
hits (no mirror) and mirrored hits that tie with a read's own query hits.  Its buckets sit on both sides of the warp tier
(256 hits) and of the CTA tier (16 384)."""
import ctypes as C

import numpy as np
import pytest

from miniasm_b200 import capi, synth
from miniasm_b200.capi import HIT_DT, SUB_DT
from miniasm_b200.pipeline import Pipeline

pytestmark = pytest.mark.gpu

# query lines of the hub reads
HUBS = [3, 100, 240, 256, 257, 1000, 8000, 16000, 16384, 16385, 20000]


def masked(h):
    h = h.copy()
    h["bl_del"] &= 0x7fffffff      # ma_hit_t::del is never written by the reference (uninitialised heap bit)
    return h


def write_mixed_paf(path):
    rng = np.random.default_rng(73)
    lines = []

    def line(q, ql, qs, qe, rev, t, tl, ts, te, ml, bl):
        f = [q, ql, qs, qe, rev, t, tl, ts, te, ml]
        if bl is not None:
            f.append(bl)
        s = "\t".join(map(str, f))
        if bl is not None and rng.integers(0, 3) == 0:
            s += "\tNM:i:0"
        lines.append(s + "\n")

    for k, n in enumerate(HUBS):
        hub = f"h{k}"
        for j in range(n):
            qs = int(rng.integers(0, 6)) * 100
            kind = rng.integers(0, 20)
            bl = None if kind == 3 else 5000 + j % 11                       # 10 fields: bl of the closest earlier 11-field line
            if kind == 0:                                                 # dropped: span below min_span
                line(hub, 12000, qs, qs + 1000, "+", f"t{rng.integers(0, 3000)}", 11000, 0, 1000, 900, bl)
            elif kind == 1:                                               # dropped: ml below min_match
                line(hub, 12000, qs, qs + 5000, "-", f"t{rng.integers(0, 3000)}", 11000, 0, 5000, 50, bl)
            elif kind == 2:                                               # self hit: one hit, no mirror
                line(hub, 12000, qs, qs + 5000, "-", hub, 12000, qs, qs + 5000, 900 + j % 7, bl)
            elif kind in (4, 5):                                          # the hub as target: a mirrored hit tying with its own
                ts = int(rng.integers(0, 6)) * 100
                line(f"t{rng.integers(0, 3000)}", 11000, 200, 5200, "+-"[j & 1], hub, 12000, ts, ts + 5000, 900 + j % 5, bl)
            else:
                ts = int(rng.integers(0, 4)) * 50
                line(hub, 12000, qs, qs + 5000, "+-"[j & 1], f"t{rng.integers(0, 3000)}", 11000, ts, ts + 5000, 900 + j % 7, bl)
        for c in range(3):                                                # short reads clearly inside the hub (dropped by -R)
            line(hub, 12000, 4000, 7000, "+", f"s{k}_{c}", 3000, 0, 3000, 2900, 3000)
    rng.shuffle(lines)
    with open(path, "w") as f:
        f.writelines(lines)
    return path


@pytest.fixture(scope="module")
def pafs(paf_dir):
    return {"mixed": write_mixed_paf(f"{paf_dir}/bucket_mixed.paf"),
            "nocont": synth.generate("-n 4000 -l 2000 -L 30000 -c 30 -j 100 -s 41", f"{paf_dir}/bucket_nocont.paf")}


def port_hits(port, paf, nocont=False):
    p = Pipeline(port, paf)
    excl = None
    if nocont:
        o = p.opt
        excl = port.ma_hit_no_cont(p.paf, o.min_span, o.min_match, o.max_hang, o.int_frac)
    p.d, n = port.sd_init(), C.c_size_t(0)
    p.hits = port.ma_hit_read(p.paf, p.opt.min_span, p.opt.min_match, p.d, C.byref(n), 1, excl)
    p.n_hits = n.value
    h = masked(p.hits_np())
    sub = p.sub1().sub_np().copy()
    p.free()
    if excl:
        port.sd_destroy(excl)
    return h, sub


def fused(prod, paf, how):
    """how: "ingest", "load_ingest_text", "sharded" (one rank) or "nocont" (-R).  Returns the hits and, for the single-GPU
    routes, ma_hit_sub's table computed on the bounds the sort left."""
    data = open(paf, "rb").read()
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    if how == "load_ingest_text":
        assert prod.mab_load_ingest_text(ctx, data, len(data), opt.min_span, opt.min_match, 1) == 0
    else:
        assert prod.mab_load_paf_text(ctx, data, len(data)) == 0
        if how == "sharded":
            assert prod.mab_shard_init(ctx, 0, 1, None) == 0
            prod.mab_ingest_sharded(ctx, opt.min_span, opt.min_match, 1)
        elif how == "nocont":
            prod.mab_ingest_nocont(ctx, opt.min_span, opt.min_match, 1, opt.max_hang, opt.int_frac)
        else:
            prod.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    n = C.c_size_t(0)
    hp = prod.mab_export_hits(ctx, C.byref(n))
    hits = masked(capi.np_from_ptr(hp, n.value, HIT_DT))
    capi.c_free(hp)
    sub = None
    if how != "sharded":
        prod.mab_select(ctx, C.byref(opt), 0, 0, 2)
        d = prod.mab_export_dict(ctx)
        sp = prod.mab_export_sub(ctx)
        sub = capi.np_from_ptr(sp, d.contents.n_seq, SUB_DT).copy()
        capi.c_free(sp), prod.sd_destroy(d)
    prod.mab_destroy(ctx)
    return hits, sub


def test_mixed_paf_reaches_every_case(pafs, port):
    h, _ = port_hits(port, pafs["mixed"])
    per_read = np.bincount((h["qns"] >> np.uint64(32)).astype(np.int64))
    assert ((per_read > 0) & (per_read <= 256)).any() and ((per_read > 256) & (per_read <= 16384)).any() and per_read.max() > 16384
    q, t = (h["qns"] >> np.uint64(32)).astype(np.int64), h["tn"].astype(np.int64)
    assert (q == t).any()                                                 # self hits
    _, runs = np.unique(h["qns"], return_counts=True)
    assert runs.max() > 1000
    with open(pafs["mixed"]) as f:
        nf = [ln.count("\t") + 1 for ln in f]
    assert 10 in nf and 11 in nf and 12 in nf


@pytest.mark.parametrize("how", ["ingest", "load_ingest_text", "sharded"])
def test_bucket_emit_matches_port(how, pafs, port, prod):
    want_h, want_sub = port_hits(port, pafs["mixed"])
    got_h, got_sub = fused(prod, pafs["mixed"], how)
    assert len(got_h) == len(want_h) and np.array_equal(got_h, want_h)
    if got_sub is not None:
        assert np.array_equal(got_sub, want_sub)


@pytest.mark.parametrize("name", ["mixed", "nocont"])
def test_bucket_emit_nocont_matches_port(name, pafs, port, prod):
    want_h, want_sub = port_hits(port, pafs[name], nocont=True)
    got_h, got_sub = fused(prod, pafs[name], "nocont")
    assert len(got_h) == len(want_h) and np.array_equal(got_h, want_h)
    assert np.array_equal(got_sub, want_sub)


def test_dropin_hit_read_matches_port(pafs, port, prod):
    """The drop-in ma_hit_read uploads the hits and sorts them with dh_sort (input position as the ordinal)."""
    p = Pipeline(prod, pafs["mixed"]).read()
    got = masked(p.hits_np())
    p.free()
    want, _ = port_hits(port, pafs["mixed"])
    assert np.array_equal(got, want)
