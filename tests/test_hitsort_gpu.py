"""The hit sort (ma_hit_sort, hit.c:19-22) keeps ties in input order: the hits must come out exactly as the oracle port's
stable merge sort leaves them, element for element, not merely as some order by (qid, qs).  Ties decide the GFA on
tie-heavy sets.  Also checked: ma_hit_sub with the per-read bounds the sort hands over and after a compaction dropped them."""
import ctypes as C

import numpy as np
import pytest

from miniasm_b200 import capi, synth
from miniasm_b200.capi import HIT_DT, SUB_DT
from miniasm_b200.pipeline import Pipeline

pytestmark = pytest.mark.gpu

SETS = ["tiny_exact", "shuffled", "chaos", "skew_small"]
# per-read bucket sizes around the warp tier (256 hits), the CTA tier (16384) and beyond it
SIZES = [1, 2, 31, 32, 33, 255, 256, 257, 700, 16384, 16385, 20000]


def masked(h):
    h = h.copy()
    h["bl_del"] &= 0x7fffffff      # ma_hit_t::del is never written by the reference (uninitialised heap bit)
    return h


def write_tie_paf(path):
    """Query reads with SIZES[k] lines each, query starts from a handful of values (long runs of equal (qid, qs)), targets
    from a pool of 3000 reads (each gets mirrored hits), lines shuffled."""
    rng = np.random.default_rng(21)
    lines = []
    for k, n in enumerate(SIZES):
        qs = rng.integers(0, 6, size=n) * 100
        tgt = rng.integers(0, 3000, size=n)
        ts = rng.integers(0, 4, size=n) * 50
        for j in range(n):
            qe, te = int(qs[j]) + 5000, int(ts[j]) + 5000
            lines.append(f"q{k}\t12000\t{qs[j]}\t{qe}\t{'+-'[j & 1]}\tt{tgt[j]}\t11000\t{ts[j]}\t{te}\t{900 + j % 7}\t5000\t255\n")
    rng.shuffle(lines)
    with open(path, "w") as f:
        f.writelines(lines)
    return path


@pytest.fixture(scope="module")
def pafs(paf_dir):
    out = {name: synth.generate(name, f"{paf_dir}/{name}.paf") for name in SETS}
    out["ties"] = write_tie_paf(f"{paf_dir}/ties.paf")
    return out


def port_hits(port, paf):
    p = Pipeline(port, paf).read()
    h = masked(p.hits_np())
    p.free()
    return h


def fused_hits(prod, paf, stream):
    data = open(paf, "rb").read()
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    if stream:
        assert prod.mab_load_ingest_text(ctx, data, len(data), opt.min_span, opt.min_match, 1) == 0
    else:
        assert prod.mab_load_paf_text(ctx, data, len(data)) == 0
        prod.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    n = C.c_size_t(0)
    hp = prod.mab_export_hits(ctx, C.byref(n))
    h = masked(capi.np_from_ptr(hp, n.value, HIT_DT))
    capi.c_free(hp)
    prod.mab_destroy(ctx)
    return h


@pytest.mark.parametrize("stream", [False, True], ids=["ingest", "load_ingest_text"])
@pytest.mark.parametrize("name", SETS + ["ties"])
def test_fused_ingest_order(name, stream, pafs, port, prod):
    want = port_hits(port, pafs[name])
    got = fused_hits(prod, pafs[name], stream)
    assert len(got) == len(want) and np.array_equal(got, want)


def test_tie_paf_reaches_every_tier(pafs, port):
    """The hand-made file really has buckets on both sides of both limits and long runs of equal keys."""
    h = port_hits(port, pafs["ties"])
    per_read = np.bincount((h["qns"] >> np.uint64(32)).astype(np.int64))
    assert per_read.max() > 16384 and ((per_read > 256) & (per_read <= 16384)).any() and ((per_read > 0) & (per_read <= 256)).any()
    _, runs = np.unique(h["qns"], return_counts=True)
    assert runs.max() > 1000


@pytest.mark.parametrize("name", ["shuffled", "skew_small", "ties"])
def test_dropin_hit_read_order(name, pafs, port, prod):
    """The drop-in ma_hit_read sorts uploaded hits with the generic sort (its own counting and bucketing passes)."""
    p = Pipeline(prod, pafs[name]).read()
    got = masked(p.hits_np())
    p.free()
    assert np.array_equal(got, port_hits(port, pafs[name]))


def fused_select_sub(prod, paf, stage):
    data = open(paf, "rb").read()
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    assert prod.mab_load_paf_text(ctx, data, len(data)) == 0
    prod.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    prod.mab_select(ctx, C.byref(opt), 0, 0, stage)
    d = prod.mab_export_dict(ctx)
    n_seq = d.contents.n_seq
    sp = prod.mab_export_sub(ctx)
    sub = capi.np_from_ptr(sp, n_seq, SUB_DT).copy()
    n = C.c_size_t(0)
    hp = prod.mab_export_hits(ctx, C.byref(n))
    hits = masked(capi.np_from_ptr(hp, n.value, HIT_DT))
    capi.c_free(hp), capi.c_free(sp), prod.sd_destroy(d), prod.mab_destroy(ctx)
    return sub, hits


@pytest.mark.parametrize("name", ["chaos", "skew_small", "ties"])
def test_sub_with_and_without_sort_bounds(name, pafs, port, prod):
    """Stage 2: the first ma_hit_sub runs on the bounds the sort left.  Stage 4: cut + flt compacted the hits (bounds dropped),
    so the second ma_hit_sub derives them from the hits again.  Both against the port's steps."""
    r = Pipeline(port, pafs[name]).read().sub1()
    want_sub1 = r.sub_np().copy()
    r.cut().flt().sub2_cut_merge()
    want_sub2, want_hits = r.sub_np().copy(), masked(r.hits_np())
    r.free()
    sub, _ = fused_select_sub(prod, pafs[name], 2)
    assert np.array_equal(sub, want_sub1)
    sub, hits = fused_select_sub(prod, pafs[name], 4)
    assert np.array_equal(sub, want_sub2) and np.array_equal(hits, want_hits)
