"""CPU tier: the oracle port against the unmodified reference (oracle/_ref/libminiasm_ref.so) on wild PAF files
(tests/wild_paf.py): pafgen sets with negative columns, columns of 2^31 and more, starts past ends, ends past lengths, lengths
that disagree between lines, reads longer than 2^31, 10-field lines and self lines.  Both run main.c:108-199 step by step under
each read-selection mode (default, -1, -2, -1 -2) and under -R; the dictionary, every interval table, the hits (del bit
masked, canonical order), the graph after ma_sg_gen and after each cleaning call, and the GFA must agree.

ma_sg_gen classifies each hit with the 32-bit read lengths `sub.e - sub.s` (or the dictionary length without a selection,
asm.c:23-24), not the 31-bit asg_seq_t::len: with -1 a second-round interval that starts below zero, and with -1 -2 a length
column of 2^31 or more, tell the two apart."""
import ctypes as C
import os

import numpy as np
import pytest

from miniasm_b200 import capi, synth
from miniasm_b200.capi import HIT_DT, SUB_DT
from miniasm_b200.pipeline import Pipeline, canon_arcs
from oracle import loaders
from tests import wild_paf

pytestmark = pytest.mark.skipif(not os.path.exists(loaders.REFERENCE_SO), reason="oracle/_ref not built (needs the reference's sources)")

BASE = "-n 800 -s 31 -j 200 -C 200000"
SEEDS = [1, 2, 3]
MODES = {"default": (False, False), "no1": (True, False), "no2": (False, True), "no12": (True, True)}


@pytest.fixture(scope="module")
def wild(built, paf_dir):
    base = synth.generate(BASE, f"{paf_dir}/wild_base.paf")
    out = {}
    for s in SEEDS:
        path = f"{paf_dir}/wild{s}.paf"
        out[s] = (path, wild_paf.make(base, path, s))
    return out


def masked_sorted(h):
    h = h.copy()
    h["bl_del"] &= 0x7fffffff
    return np.sort(h, order=list(HIT_DT.names))


def steps(lib, paf, no_first, no_second, no_cont=False):
    """main.c:108-199 one call at a time; yields (step, state) after each call."""
    p = Pipeline(lib, paf)
    o = p.opt
    excl = lib.ma_hit_no_cont(p.paf, o.min_span, o.min_match, o.max_hang, o.int_frac) if no_cont else None
    p.d, n = lib.sd_init(), C.c_size_t(0)
    p.hits = lib.ma_hit_read(p.paf, o.min_span, o.min_match, p.d, C.byref(n), 1, excl)
    p.n_hits = n.value
    d = p.d.contents
    yield "read", [[(d.seq[i].name, d.seq[i].len) for i in range(d.n_seq)], masked_sorted(p.hits_np())]
    n_seq = d.n_seq
    if not no_first:
        p.sub1()
        yield "sub1", p.sub_np().copy()
        p.cut()
        yield "cut1", masked_sorted(p.hits_np())
        p.flt()
        yield "flt", [masked_sorted(p.hits_np()), np.float32(p.cov.value)]
    if not no_second:
        sub2 = lib.ma_hit_sub(o.min_dp, o.min_iden, o.min_span // 2, p.n_hits, p.hits, n_seq)
        yield "sub2", capi.np_from_ptr(sub2, n_seq, SUB_DT).copy()
        p.n_hits = lib.ma_hit_cut(sub2, o.min_span, p.n_hits, p.hits)
        yield "cut2", masked_sorted(p.hits_np())
        if not no_first:
            lib.ma_sub_merge(n_seq, p.sub, sub2)
            capi.c_free(sub2)
        else:
            p.sub = sub2
        yield "merge", p.sub_np().copy()
        p.contained()
        d = p.d.contents
        yield "contained", [p.names(), p.sub_np().copy(), masked_sorted(p.hits_np())]
    p.sg_gen()

    def graph():
        arcs, seq, _, _, _ = lib.read_graph(p.sg)
        return [canon_arcs(arcs), seq.copy()]
    yield "sg_gen", graph()
    yield "clean", p.sg
    p.clean().ug_gen()
    yield "gfa", p.gfa()
    p.free()
    if excl:
        lib.sd_destroy(excl)


def same_state(a, b):
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(same_state(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)
    return a == b


def clean_calls(o):
    """The cleaning calls of main.c:156-188; a call after which main.c goes on only if it removed something is marked."""
    calls = [("asg_arc_del_trans", (o.gap_fuzz,), False), ("asg_cut_tip", (o.max_ext,), False), ("asg_pop_bubble", (o.bub_dist,), False)]
    for i in range(o.n_rounds + 1):
        r = np.float32(o.min_ovlp_drop_ratio) + (np.float32(o.max_ovlp_drop_ratio) - np.float32(o.min_ovlp_drop_ratio)) \
            / np.float32(o.n_rounds) * np.float32(i)
        calls += [("asg_arc_del_short", (float(r),), False), ("asg_cut_tip", (o.max_ext,), True), ("asg_pop_bubble", (o.bub_dist,), True)]
    calls += [("asg_cut_internal", (1,), False), ("asg_cut_biloop", (o.max_ext,), False), ("asg_cut_tip", (o.max_ext,), False),
              ("asg_pop_bubble", (o.bub_dist,), False)]
    calls += [("asg_arc_del_short", (o.final_ovlp_drop_ratio,), False), ("asg_cut_tip", (o.max_ext,), True), ("asg_pop_bubble", (o.bub_dist,), True)]
    return calls


def clean_stepwise(ref, port, sg):
    """Each cleaning call on both sides from the same pre-state (a copy of the port's graph): the order of tied arcs, which the
    reference's unstable sort decides, then cannot move counts between calls."""
    g = port.clone_graph(sg)
    o, last = port.default_opt(), 1
    for fn, args, cond in clean_calls(o):
        if cond and last == 0:
            continue

        def run(lib):
            h = lib.clone_graph(g) if lib is port else lib.make_graph(*port.read_graph(g)[:2], *port.read_graph(g)[3:])
            if lib is not port and port.read_graph(g)[2] is not None:
                h.contents.idx = capi.c_malloc_copy(port.read_graph(g)[2])
            k = getattr(lib, fn)(h, *args)
            a, s, i, srt, symm = lib.read_graph(h)
            out = [k, a.copy(), s.copy(), None if i is None else i.copy(), srt, symm]
            lib.asg_destroy(h)
            return out
        got, want = run(port), run(ref)
        assert same_state(got, want), f"{fn}{args} differs from the reference"
        k = getattr(port, fn)(g, *args)
        if fn == "asg_arc_del_short":
            last = k
    port.asg_destroy(g)


def compare(ref, port, paf, **kw):
    n = 0
    for (sr, vr), (sp, vp) in zip(steps(ref, paf, **kw), steps(port, paf, **kw)):
        assert sr == sp
        if sp == "clean":
            clean_stepwise(ref, port, vp)
        else:
            assert same_state(vp, vr), f"{sp} (step {n}) differs from the reference"
        n += 1
    return n


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("mode", list(MODES))
def test_wild_port_matches_reference(mode, seed, wild, ref, port):
    no_first, no_second = MODES[mode]
    assert compare(ref, port, wild[seed][0], no_first=no_first, no_second=no_second) == 11 - 3 * no_first - 4 * no_second


@pytest.mark.parametrize("seed", SEEDS)
def test_wild_no_cont(seed, wild, ref, port):
    assert compare(ref, port, wild[seed][0], no_first=False, no_second=False, no_cont=True) == 11


def test_wild_reaches_every_class(wild, port):
    """Every class was applied; a hit of a read longer than 2^31 reaches ma_sg_gen under -1 -2; a second-round interval that
    starts below zero (a negative 32-bit length) exists under -1 and survives to ma_sg_gen; the selection keeps thousands of hits."""
    for seed, (paf, counts) in wild.items():
        assert all(counts[c] > 0 for c in wild_paf.CLASSES), counts
        p = Pipeline(port, paf).read()
        lens = p.seq_lens()
        assert (lens >= 1 << 31).sum() >= 3
        q = (p.hits_np()["qns"] >> np.uint64(32)).astype(np.int64)
        assert (lens[q] >= 1 << 31).sum() > 0                      # -1 -2 hands these to ma_sg_gen as they are
        o, n_seq = p.opt, p.d.contents.n_seq
        sub2 = port.ma_hit_sub(o.min_dp, o.min_iden, o.min_span // 2, p.n_hits, p.hits, n_seq)
        s2 = capi.np_from_ptr(sub2, n_seq, SUB_DT).copy()
        p.n_hits = port.ma_hit_cut(sub2, o.min_span, p.n_hits, p.hits)
        p.sub = sub2
        live = (s2["s_del"] & np.uint32(0x80000000)) == 0
        ln32 = (s2["e"] - (s2["s_del"] & np.uint32(0x7fffffff))).astype(np.uint32)
        wrapped = live & (ln32 >= np.uint32(1 << 31))
        assert wrapped.any()
        q = (p.hits_np()["qns"] >> np.uint64(32)).astype(np.int64)
        assert wrapped[q].any()                                    # ... and it still has hits after the second cut
        p.contained()
        assert p.n_hits > 1000
        p.free()
        r = Pipeline(port, paf).read().select()
        assert r.n_hits > 1000
        r.free()
