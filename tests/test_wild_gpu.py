"""GPU tier on wild PAF files (tests/wild_paf.py) and wild hit arrays (tests/test_hitrules_cpu.fuzz): negative columns, columns of
2^31 and more, starts past ends, ends past lengths, lengths that disagree between lines, reads longer than 2^31, 10-field lines,
self lines.  Under -1 and -1 -2 ma_sg_gen classifies hits with 32-bit read lengths of 2^31 or more (asm.c:23-24), which the
31-bit asg_seq_t::len cannot hold; the graph kernels take them from the 32-bit length array instead.

* the command line against the reference (stored digests, tests/refgold.py): outputs and counters of every selection mode, the
  -S stage dumps in paf, bed, sg and ug;
* the fused API against the oracle port: mab_select under each mode and step path, mab_layout stage by stage, mab_load_hits,
  the one-rank sharded path;
* the drop-in entry points on fuzzed hits with interval lengths of 2^31 and more, against the reference;
* ma_hit_sub's warp and CTA tiers on groups whose starts wrap past 2^32 once end_clip is added."""
import ctypes as C

import numpy as np
import pytest

from miniasm_b200 import capi, synth
from miniasm_b200.capi import HIT_DT, SUB_DT
from miniasm_b200.pipeline import Pipeline, canon_arcs
from tests import wild_paf
from tests.test_cli_gpu import OURS, REF, _counters, outcome, run
from tests.test_hitrules_cpu import fuzz

pytestmark = pytest.mark.gpu

BASE = "-n 800 -s 31 -j 200 -C 200000"
SEEDS = [1, 2, 3]
MODES = {"default": (0, 0), "no1": (1, 0), "no2": (0, 1), "no12": (1, 1)}


@pytest.fixture(scope="module")
def wild(built, paf_dir):
    base = synth.generate(BASE, f"{paf_dir}/wild_base.paf")
    return {s: wild_paf.make(base, f"{paf_dir}/wild{s}.paf", s) and f"{paf_dir}/wild{s}.paf" for s in SEEDS}


def same(gold, args, exact=True, counters=False):
    rc, out, err = run(OURS, args)
    assert rc == 0, err.decode()[-2000:]
    gold.cli("exact" if exact else "sorted", args, outcome(rc, out, exact), lambda: outcome(*run(REF, args)[:2], exact))
    if counters:
        gold.cli("counters, reduced + asymmetric as a sum", args, norm(_counters(err)), lambda: norm(_counters(run(REF, args)[2])))


def norm(lines):
    """The counters, with asg_arc_del_trans's count and the asymmetric-arc count of the asg_symm inside it as their sum: which of
    two tied arcs the reference's unstable sort puts first can move an arc from one to the other, and the graph after asg_symm is
    the same (DESIGN.md "Tie order", tests/test_cli_gpu.py::test_bubble_dense_300k)."""
    i = next(k for k, x in enumerate(lines) if "transitively reduced" in x)
    j = next(k for k, x in enumerate(lines) if k > i and "asymmetric arcs" in x)
    num = lambda x: int([t for t in x.split() if t.isdigit()][0])
    return [x for k, x in enumerate(lines) if k not in (i, j)], num(lines[i]) + num(lines[j])


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("opts", [[], ["-1"], ["-2"], ["-1", "-2"], ["-R"], ["-c", "2", "-e", "2"]],
                         ids=["default", "no1", "no2", "no12", "R", "c2e2"])
def test_cli_modes(opts, seed, wild, gold):
    same(gold, opts + [wild[seed]], counters=True)


@pytest.mark.parametrize("seed", SEEDS)
def test_cli_stage_dumps(seed, wild, gold):
    paf = wild[seed]
    for stage in ("2", "3", "4", "5"):
        same(gold, ["-S", stage, "-p", "paf", paf], exact=False)
    for stage in ("2", "3", "4", "5", "100"):
        same(gold, ["-S", stage, "-p", "bed", paf])
    for stage in (1, 5, 6, 7, 9, 10, 11):
        same(gold, ["-S", str(stage), "-p", "sg", paf], exact=stage >= 6)
    same(gold, ["-p", "ug", paf])
    # the raw graph of -1 and -1 -2, where the 32-bit lengths decide (-p paf / bed would read a NULL sub in the reference under -1 -2)
    same(gold, ["-1", "-S", "5", "-p", "sg", paf], exact=False)
    same(gold, ["-1", "-2", "-S", "5", "-p", "sg", paf], exact=False)


# ---- fused API against the oracle port ------------------------------------------------------------------------------------
def masked_sorted(h):
    h = h.copy()
    h["bl_del"] &= 0x7fffffff
    return np.sort(h, order=list(HIT_DT.names))


def port_run(port, paf, no_first, no_second, stage):
    """main.c:116-142 with -S stage on the port; the selection's state, then the raw graph and the GFA."""
    p = Pipeline(port, paf).read()
    o, n_seq = p.opt, p.d.contents.n_seq
    if not no_first:
        if stage >= 2:
            p.sub1().cut()
        if stage >= 3:
            p.flt()
    if not no_second:
        if stage >= 4:
            sub2 = port.ma_hit_sub(o.min_dp, o.min_iden, o.min_span // 2, p.n_hits, p.hits, n_seq)
            p.n_hits = port.ma_hit_cut(sub2, o.min_span, p.n_hits, p.hits)
            if not no_first:
                port.ma_sub_merge(n_seq, p.sub, sub2)
                capi.c_free(sub2)
            else:
                p.sub = sub2
        if stage >= 5:
            p.contained()
    sel = {"names": p.names(), "hits": masked_sorted(p.hits_np()), "sub": None if not p.sub else p.sub_np().copy()}
    p.sg_gen()
    a, s, i, srt, _ = p.graph_np()
    raw = [s.copy(), canon_arcs(a)]
    p.clean().ug_gen()
    gfa = p.gfa()
    p.free()
    return sel, raw, gfa


def prod_select(prod, paf, no_first, no_second, stage, how="ingest"):
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    if how == "hits":
        from oracle import loaders
        q = Pipeline(loaders.load_oracle_port(), paf).read()
        assert prod.mab_load_hits(ctx, q.hits, q.n_hits, q.d) == 0
        q.free()
    else:
        data = open(paf, "rb").read()
        assert prod.mab_load_paf_text(ctx, data, len(data)) == 0
        if how == "sharded":
            assert prod.mab_shard_init(ctx, 0, 1, None) == 0
            prod.mab_ingest_sharded(ctx, opt.min_span, opt.min_match, 1)
        else:
            prod.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    if how == "sharded":
        prod.mab_select_sharded(ctx, C.byref(opt))
    else:
        prod.mab_select(ctx, C.byref(opt), no_first, no_second, stage)
    return ctx, opt


def prod_state(prod, ctx):
    d = prod.mab_export_dict(ctx)
    n_seq = d.contents.n_seq
    names = [d.contents.seq[i].name for i in range(n_seq)]
    n = C.c_size_t(0)
    hp = prod.mab_export_hits(ctx, C.byref(n))
    hits = masked_sorted(capi.np_from_ptr(hp, n.value, HIT_DT))
    sp = prod.mab_export_sub(ctx)
    sub = capi.np_from_ptr(sp, n_seq, SUB_DT).copy() if sp else None
    capi.c_free(hp), capi.c_free(sp), prod.sd_destroy(d)
    return {"names": names, "hits": hits, "sub": sub}


def prod_layout(prod, ctx, opt):
    prod.mab_layout(ctx, C.byref(opt), 5)
    g = prod.mab_export_sg(ctx)
    a, s, _, _, _ = prod.read_graph(g)
    raw = [s.copy(), canon_arcs(a)]
    prod.asg_destroy(g)
    prod.mab_layout(ctx, C.byref(opt), 100)
    prod.mab_unitigs(ctx)
    d, sub, ug = prod.mab_export_dict(ctx), prod.mab_export_sub(ctx), prod.mab_export_ug(ctx)
    gfa = prod.print_to_string("ma_ug_print", ug, d, sub)
    prod.ma_ug_destroy(ug), capi.c_free(sub), prod.sd_destroy(d)
    return raw, gfa


def check_sel(got, want):
    assert got["names"] == want["names"]
    assert len(got["hits"]) == len(want["hits"]) and np.array_equal(got["hits"], want["hits"])
    if want["sub"] is not None:
        assert got["sub"] is not None and np.array_equal(got["sub"], want["sub"])


def check_raw(got, want):
    assert np.array_equal(got[0], want[0])                          # lengths (31 bits) and del bits
    assert len(got[1]) == len(want[1]) and np.array_equal(got[1], want[1])


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("mode", list(MODES))
def test_fused_matches_port(mode, seed, wild, port, prod):
    no_first, no_second = MODES[mode]
    sel, raw, gfa = port_run(port, wild[seed], no_first, no_second, 100)
    ctx, opt = prod_select(prod, wild[seed], no_first, no_second, 100)
    check_sel(prod_state(prod, ctx), sel)
    got_raw, got_gfa = prod_layout(prod, ctx, opt)
    check_raw(got_raw, raw)
    assert got_gfa == gfa
    prod.mab_destroy(ctx)


@pytest.mark.parametrize("stage", [2, 3, 4, 5])
def test_fused_step_paths(stage, wild, port, prod):
    """The step paths of mab_select (-S 2..5): the selection's state and the graph built on it."""
    sel, raw, gfa = port_run(port, wild[1], 0, 0, stage)
    ctx, opt = prod_select(prod, wild[1], 0, 0, stage)
    check_sel(prod_state(prod, ctx), sel)
    got_raw, got_gfa = prod_layout(prod, ctx, opt)
    check_raw(got_raw, raw)
    assert got_gfa == gfa
    prod.mab_destroy(ctx)


@pytest.mark.parametrize("mode", ["default", "no1", "no12"])
def test_fused_from_loaded_hits(mode, wild, port, prod):
    no_first, no_second = MODES[mode]
    sel, raw, gfa = port_run(port, wild[2], no_first, no_second, 100)
    ctx, opt = prod_select(prod, wild[2], no_first, no_second, 100, how="hits")
    check_sel(prod_state(prod, ctx), sel)
    got_raw, got_gfa = prod_layout(prod, ctx, opt)
    check_raw(got_raw, raw)
    assert got_gfa == gfa
    prod.mab_destroy(ctx)


@pytest.mark.parametrize("seed", SEEDS)
def test_fused_sharded_one_rank(seed, wild, port, prod):
    sel, _, gfa = port_run(port, wild[seed], 0, 0, 100)
    ctx, opt = prod_select(prod, wild[seed], 0, 0, 100, how="sharded")
    check_sel(prod_state(prod, ctx), sel)
    prod.mab_layout_sharded(ctx, C.byref(opt))
    prod.mab_unitigs(ctx)
    d, sub, ug = prod.mab_export_dict(ctx), prod.mab_export_sub(ctx), prod.mab_export_ug(ctx)
    assert prod.print_to_string("ma_ug_print", ug, d, sub) == gfa
    prod.ma_ug_destroy(ug), capi.c_free(sub), prod.sd_destroy(d), prod.mab_destroy(ctx)


# ---- drop-in entry points on fuzzed hits ----------------------------------------------------------------------------------
def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _dict(lib, lens):
    d = lib.sd_init()
    for i, ln in enumerate(lens):
        lib.sd_put(d, f"r{i}".encode(), int(ln))
    return d


def dropin(lib, seed, wild):
    """Every drop-in step on one fuzzed interval table and hit array; what each step returns."""
    sub, h = fuzz(600 + seed, wild=wild)
    n_seq = len(sub)
    o = lib.default_opt()
    out = []
    for clip in (0, 1000):
        hp = capi.c_malloc_copy(h)
        s = lib.ma_hit_sub(o.min_dp, o.min_iden, clip, len(h), hp, n_seq)
        out.append(capi.np_from_ptr(s, n_seq, SUB_DT).copy())
        capi.c_free(s), capi.c_free(hp)
    a = h.copy()
    n = lib.ma_hit_cut(_ptr(sub), 1000, len(a), _ptr(a))
    out.append(a[:n].copy())
    a = h.copy()
    cov = C.c_float(0)
    n = lib.ma_hit_flt(_ptr(sub), 1500, 1000, len(a), _ptr(a), C.byref(cov))
    out += [a[:n].copy(), np.float32(cov.value)]
    len32 = (sub["e"] - (sub["s_del"] & np.uint32(0x7fffffff))).astype(np.uint32)
    for with_sub in (True, False):
        # without sub the dictionary lengths are the 32-bit ones (a read of 2^31 or more where the interval wrapped)
        d = _dict(lib, np.full(n_seq, 20000) if with_sub else len32)
        g = lib.ma_sg_gen(C.byref(o), d, _ptr(sub) if with_sub else None, len(h), _ptr(h))
        arcs, seq, _, _, _ = lib.read_graph(g)
        out += [canon_arcs(arcs), seq.copy()]
        lib.asg_destroy(g), lib.sd_destroy(d)
    d = _dict(lib, np.full(n_seq, 20000))
    s2, a = sub.copy(), h.copy()
    n = lib.ma_hit_contained(C.byref(o), d, _ptr(s2), len(a), _ptr(a))
    out += [np.sort(a[:n], order=list(HIT_DT.names)), s2[:d.contents.n_seq].copy(), [d.contents.seq[i].name for i in range(d.contents.n_seq)]]
    lib.sd_destroy(d)
    return out


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("wild", [True, "long"], ids=["wild", "long"])
def test_dropin_fuzz(seed, wild, prod, ref, gold):
    for k, x in enumerate(dropin(prod, seed, wild)):
        gold.expect(x, lambda k=k: dropin(ref, seed, wild)[k])


# ---- ma_hit_sub tiers with starts that wrap past 2^32 ----------------------------------------------------------------------
def wrap_group_hits(n, max_coord, seed):
    """One read (id 0) with n hits; a third of their starts lie within 1000 of 2^32, so qs + end_clip wraps to below 1000, and
    the other coordinates stay below max_coord (the key range picks the CTA tier's counting or bitonic path)."""
    rng = np.random.default_rng(seed + n)
    qs = rng.integers(0, max_coord // 2, n).astype(np.uint64)
    qe = np.minimum(qs + rng.integers(2500, 8000, n).astype(np.uint64), np.uint64(max_coord - 1))
    far = rng.random(n) < 1 / 3
    qs[far] = (1 << 32) - rng.integers(1, 1000, int(far.sum())).astype(np.uint64)
    h = np.zeros(n, dtype=HIT_DT)
    h["qns"], h["qe"] = qs, qe
    h["tn"] = 1 + np.arange(n) % 7
    span = (qe - qs) & np.uint64(0xffffffff)
    h["ml_rev"], h["bl_del"] = (span // 2).astype(np.uint32) & np.uint32(0x7fffffff), span.astype(np.uint32) & np.uint32(0x7fffffff)
    return h[np.argsort(h["qns"], kind="stable")]


@pytest.mark.parametrize("n", [3, 256, 257, 16384, 16385])
@pytest.mark.parametrize("max_coord", [30000, 1 << 20], ids=["counting", "bitonic"])
@pytest.mark.parametrize("clip", [0, 1000])
def test_sub_tiers_wrapping(n, max_coord, clip, port, prod):
    h = wrap_group_hits(n, max_coord, 7)
    o = prod.default_opt()
    subs = []
    for lib in (prod, port):
        p = capi.c_malloc_copy(h)
        s = lib.ma_hit_sub(1 if n == 3 else o.min_dp, o.min_iden, clip, len(h), p, 8)
        subs.append(capi.np_from_ptr(s, 8, SUB_DT).copy())
        capi.c_free(s), capi.c_free(p)
    assert np.array_equal(subs[0], subs[1])
    if clip:
        assert subs[1]["s_del"][0] & np.uint32(0x80000000) == 0
