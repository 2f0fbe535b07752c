"""The default read selection (mab_select with stage 100) runs as per-read passes over the hit buckets.  Its results must be
exactly what the oracle port's step functions give: the merged interval table, the surviving hits in order (del bit masked),
names, read and hit counts, and the [M::ma_hit_*] counters printed at verbose 3.  Inputs: the synthetic sets, and a hand-made
file whose reads sit on both sides of every tier limit after filtering and that has hits dropped by each step."""
import ctypes as C
import re

import numpy as np
import pytest

from miniasm_b200 import capi, synth
from miniasm_b200.capi import HIT_DT, SUB_DT
from miniasm_b200.pipeline import Pipeline

pytestmark = pytest.mark.gpu

SETS = ["tiny_exact", "jitter30", "varlen300", "bubbles800", "chaos", "chaos_small", "shuffled", "skew_small", "lowcov", "c1_ecoli_like"]
# post-filter hit counts of the hub reads: both sides of the warp tier's chunk (32), of the warp tier (256) and of the CTA tier (16384)
TIERS = [32, 33, 256, 257, 16384, 16385]
DEL = np.uint32(0x80000000)


def masked(h):
    h = h.copy()
    h["bl_del"] &= 0x7fffffff      # ma_hit_t::del is never written by the reference (uninitialised heap bit)
    return h


def write_tiers_paf(path):
    """Hub reads (20 kb) holding 6 kb partner reads, each partner in three or four identical lines so that its own depth
    reaches min_dp; hub k ends up with TIERS[k] hits after filtering.  Each hub also has one internal match with a read that a
    carrier hub holds (dropped by ma_hit_flt), and read z has its only hits with three reads of depth one (all dropped by
    ma_hit_cut).  Partners are contained in their hubs, so ma_hit_contained drops them; a chain of overlapping reads keeps
    some hits to the end."""
    lines = []

    def line(q, ql, qs, qe, t, tl, ts, te):
        lines.append(f"{q}\t{ql}\t{qs}\t{qe}\t+\t{t}\t{tl}\t{ts}\t{te}\t{(qe - qs) // 2}\t{qe - qs}\t255\n")

    for k, want in enumerate(TIERS):
        n_part = want // 3
        for j in range(n_part):
            x = round(j * 14000 / (n_part - 1))
            for _ in range(3 + (j < want % 3)):
                line(f"p{k}_{j}", 6000, 0, 6000, f"h{k}", 20000, x, x + 6000)
        for _ in range(3):
            line(f"i{k}", 8000, 0, 8000, f"c{k}", 20000, 0, 8000)
        line(f"h{k}", 20000, 5000, 8000, f"i{k}", 8000, 2000, 5000)
    for j in range(3):
        line("z", 6000, 0, 6000, f"l{j}", 6000, 0, 6000)
    for i in range(7):   # a chain of dovetails: its inner reads and their hits survive the selection
        for _ in range(3):
            line(f"a{i}", 10000, 3000, 10000, f"a{i + 1}", 10000, 0, 7000)
    with open(path, "w") as f:
        f.writelines(lines)
    return path


@pytest.fixture(scope="module")
def pafs(paf_dir):
    out = {name: synth.generate(name, f"{paf_dir}/{name}.paf") for name in SETS}
    out["tiers"] = write_tiers_paf(f"{paf_dir}/tiers.paf")
    return out


def n_kept(sub):
    return int(((sub["s_del"] & DEL) == 0).sum() - ((sub["s_del"] == 0) & (sub["e"] == 0)).sum())


def port_select(port, paf):
    """The port's steps, and the [M::ma_hit_*] lines the reference prints for them."""
    p = Pipeline(port, paf).read()
    o, n_seq = p.opt, p.d.contents.n_seq
    p.sub1()
    lines = [f"ma_hit_sub: {n_kept(p.sub_np())} query sequences remain after sub"]
    p.cut()
    lines.append(f"ma_hit_cut: {p.n_hits} hits remain after cut")
    p.flt()
    lines.append(f"ma_hit_flt: {p.n_hits} hits remain after filtering; crude coverage after filtering: {p.cov.value:.2f}")
    s2 = port.ma_hit_sub(o.min_dp, o.min_iden, o.min_span // 2, p.n_hits, p.hits, n_seq)
    lines.append(f"ma_hit_sub: {n_kept(capi.np_from_ptr(s2, n_seq, SUB_DT))} query sequences remain after sub")
    capi.c_free(s2)
    p.sub2_cut_merge()
    lines.append(f"ma_hit_cut: {p.n_hits} hits remain after cut")
    p.contained()
    n_seq = p.d.contents.n_seq
    lines.append(f"ma_hit_contained: {n_seq} sequences and {p.n_hits} hits remain after containment removal")
    out = {"sub": p.sub_np().copy(), "hits": masked(p.hits_np()), "names": p.names(), "n_seq": n_seq, "lines": lines}
    p.free()
    return out


def counter_lines(err):
    return [f"{m.group(1)}: {m.group(2)}" for m in re.finditer(r"^\[M::(ma_hit_\w+)::[^\]]*\] (.*)$", err, re.M)]


def fused_select(prod, port, paf, capfd, from_hits):
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    if from_hits:   # hits handed over without the sort's per-read bounds
        p = Pipeline(port, paf).read()
        assert prod.mab_load_hits(ctx, p.hits, p.n_hits, p.d) == 0
        p.free()
    else:
        data = open(paf, "rb").read()
        assert prod.mab_load_paf_text(ctx, data, len(data)) == 0
        prod.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    capfd.readouterr()
    prod.set_verbose(3)
    try:
        prod.mab_select(ctx, C.byref(opt), 0, 0, 100)
        prod.mab_sync(ctx)
    finally:
        prod.set_verbose(0)
    lines = counter_lines(capfd.readouterr().err)
    d = prod.mab_export_dict(ctx)
    n_seq = d.contents.n_seq
    names = [d.contents.seq[i].name for i in range(n_seq)]
    sp = prod.mab_export_sub(ctx)
    sub = capi.np_from_ptr(sp, n_seq, SUB_DT).copy()
    n = C.c_size_t(0)
    hp = prod.mab_export_hits(ctx, C.byref(n))
    hits = masked(capi.np_from_ptr(hp, n.value, HIT_DT))
    capi.c_free(hp), capi.c_free(sp), prod.sd_destroy(d), prod.mab_destroy(ctx)
    return {"sub": sub, "hits": hits, "names": names, "n_seq": n_seq, "lines": lines}


def check(got, want):
    assert got["lines"] == want["lines"]
    assert got["n_seq"] == want["n_seq"] and got["names"] == want["names"]
    assert np.array_equal(got["sub"], want["sub"])
    assert len(got["hits"]) == len(want["hits"]) and np.array_equal(got["hits"], want["hits"])


@pytest.mark.parametrize("name", SETS + ["tiers"])
def test_select_matches_port(name, pafs, port, prod, capfd):
    check(fused_select(prod, port, pafs[name], capfd, False), port_select(port, pafs[name]))


@pytest.mark.parametrize("name", ["chaos", "skew_small", "tiers"])
def test_select_from_loaded_hits(name, pafs, port, prod, capfd):
    check(fused_select(prod, port, pafs[name], capfd, True), port_select(port, pafs[name]))


def test_tiers_paf_reaches_every_case(pafs, port):
    """The hand-made file has reads on both sides of every tier limit after filtering, and hits dropped by the first cut, by
    the filter and by containment, including a read that loses all its hits before the second round."""
    p = Pipeline(port, pafs["tiers"]).read()
    n_seq = p.d.contents.n_seq

    def per_read():
        return np.bincount((p.hits_np()["qns"] >> np.uint64(32)).astype(np.int64), minlength=n_seq)

    before = per_read()
    p.sub1().cut()
    after_cut = per_read()
    p.flt()
    after_flt = per_read()
    assert set(TIERS) <= set(after_flt.tolist())
    assert after_cut.sum() < before.sum() and after_flt.sum() < after_cut.sum()
    assert ((before > 0) & (after_flt == 0)).any()
    n_hits = p.n_hits
    p.sub2_cut_merge().contained()
    assert p.d.contents.n_seq < n_seq and 0 < p.n_hits < n_hits
    p.free()
