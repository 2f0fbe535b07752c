"""CPU tier on layouts with repeats, inverted repeats, tandem arrays, plasmids and a heterozygous region (tests/layout_paf.py),
and on motif graphs built directly (tests/graph_fuzz.py): the oracle port step by step and the host build of
clean_fix.cuh pass by pass against the unmodified reference, and checks that each set reaches the topology it was built for."""
from collections import Counter

import numpy as np
import pytest

from miniasm_b200 import capi
from miniasm_b200.capi import DEL
from miniasm_b200.pipeline import Pipeline, canon_arcs
from tests import graph_fuzz, layout_paf
from tests.test_fix_cpu import Stepper as FixStepper, sim  # noqa: F401  (sim: the host build of clean_fix.cuh, a fixture)

SETS = list(layout_paf.SETS)
FUZZ = list(graph_fuzz.CASES)


@pytest.fixture(scope="module")
def lpafs(paf_dir):
    return {name: layout_paf.generate(name, f"{paf_dir}/lp_{name}.paf") for name in SETS}


def mask(h):
    h = h.copy()
    h["bl_del"] &= 0x7fffffff
    return h


def ratio(o, i):
    return float(np.float32(o.min_ovlp_drop_ratio) + (np.float32(o.max_ovlp_drop_ratio) - np.float32(o.min_ovlp_drop_ratio))
                 / np.float32(o.n_rounds) * np.float32(i))


def clean_passes(step, lib, g, o, max_ext=None, bub_dist=None):
    """main.c's stage (iii) after asg_arc_del_trans: `step` runs the passes under test, `lib` the arc-length filter."""
    max_ext = o.max_ext if max_ext is None else max_ext
    bub_dist = o.bub_dist if bub_dist is None else bub_dist
    step("asg_cut_tip", g, max_ext)
    step("asg_pop_bubble", g, bub_dist)
    for i in range(o.n_rounds + 1):
        if lib.asg_arc_del_short(g, ratio(o, i)):
            step("asg_cut_tip", g, max_ext)
            step("asg_pop_bubble", g, bub_dist)
    step("asg_cut_internal", g, 1)
    step("asg_cut_biloop", g, max_ext)
    step("asg_cut_tip", g, max_ext)
    step("asg_pop_bubble", g, bub_dist)
    if lib.asg_arc_del_short(g, o.final_ovlp_drop_ratio):
        step("asg_cut_tip", g, max_ext)
        step("asg_pop_bubble", g, bub_dist)


def fuzz_graph(lib, name):
    """The motif graph as ma_sg_gen leaves a graph: arcs sorted and indexed (asg_cleanup)."""
    arcs, seq, params = graph_fuzz.build(name)
    g = lib.make_graph(arcs, seq)
    lib.asg_cleanup(g)
    return g, params


@pytest.mark.parametrize("name", SETS)
def test_paf_bytes_are_pinned(name, lpafs):
    assert layout_paf.sha256(lpafs[name]) == layout_paf.SHA256[name]


@pytest.mark.parametrize("name", SETS)
def test_port_matches_reference_stepwise(name, lpafs, ref, port, gold):
    """As test_oracle_cpu.py: every step of the port from the port's own pre-state against the reference from the same one."""
    paf = lpafs[name]
    hits = lambda q: [q.names(), np.sort(mask(q.hits_np()), order=list(capi.HIT_DT.names))]
    p = Pipeline(port, paf, opt=layout_paf.opt_for(port, name)).read()

    def read_ref():
        r = Pipeline(ref, paf, opt=layout_paf.opt_for(ref, name)).read()
        out = hits(r)
        r.free()
        return out
    gold.expect(hits(p), read_ref)

    def after(lib, step, state):
        q = Pipeline(lib, paf, opt=p.opt).adopt(p)
        getattr(q, step)()
        out = state(q)
        q.free()
        return out
    state = lambda q: [q.n_hits, mask(q.hits_np()), q.sub_np(), q.names()]
    for step in ("sub1", "cut", "flt", "sub2_cut_merge", "contained"):
        gold.expect(after(port, step, state), lambda: after(ref, step, state))
        getattr(p, step)()
    sg = lambda q: (lambda a, s, i: [canon_arcs(a), s, i])(*q.graph_np()[:3])
    gold.expect(after(port, "sg_gen", sg), lambda: after(ref, "sg_gen", sg))
    p.sg_gen()

    def run(lib, fn, args):
        arcs, seq, idx, srt, symm = port.read_graph(p.sg)
        g2 = lib.make_graph(arcs, seq, srt, symm)
        if idx is not None:
            g2.contents.idx = capi.c_malloc_copy(idx)
        n = getattr(lib, fn)(g2, *args)
        out = [n, *lib.read_graph(g2)]
        lib.asg_destroy(g2)
        return out

    def step(fn, g, *args):
        gold.expect(run(port, fn, args), lambda: run(ref, fn, args))
        return getattr(port, fn)(g, *args)
    step("asg_arc_del_trans", p.sg, p.opt.gap_fuzz)
    clean_passes(step, port, p.sg, p.opt)

    def unitigs(lib):
        ug = lib.ma_ug_gen(p.sg)
        text = lib.print_to_string("ma_ug_print", ug, p.d, p.sub)
        lib.ma_ug_destroy(ug)
        return text
    gold.expect(unitigs(port), lambda: unitigs(ref))
    p.free()


@pytest.mark.parametrize("name", SETS)
def test_fixpoint_passes_on_layouts(name, lpafs, ref, sim):
    """The host build of clean_fix.cuh against the reference, pass by pass on the graph the reference built."""
    r = Pipeline(ref, lpafs[name], opt=layout_paf.opt_for(ref, name)).read().select().sg_gen()
    st = FixStepper(ref, sim)
    ref.asg_arc_del_trans(r.sg, r.opt.gap_fuzz)
    clean_passes(st.step, ref, r.sg, r.opt)
    print(name, "max sweeps per pass:", st.sweeps, "actions:", st.acted)
    r.free()


@pytest.mark.parametrize("name", FUZZ)
def test_fixpoint_passes_on_motif_graphs(name, ref, sim):
    """Each pass alone on the raw motif graph (nothing transitively reduced), then the whole stage (iii) from
    asg_arc_del_trans on, with the host build of clean_fix.cuh against the reference at every pass."""
    g, prm = fuzz_graph(ref, name)
    o = ref.default_opt()
    st = FixStepper(ref, sim)
    for fn, arg in (("asg_pop_bubble", prm["bub_dist"]), ("asg_cut_tip", prm["max_ext"]), ("asg_cut_internal", 1),
                    ("asg_cut_biloop", prm["max_ext"]), ("asg_cut_internal", prm["max_ext"])):
        h = ref.clone_graph(g)
        st.step(fn, h, arg)
        ref.asg_destroy(h)
    ref.asg_arc_del_trans(g, o.gap_fuzz)
    clean_passes(st.step, ref, g, o, prm["max_ext"], prm["bub_dist"])
    ref.asg_destroy(g)


def test_dense_graph_walk_exceeds_four_arcs_per_vertex(ref, sim):
    """The dense motif graph: the bubble walk from read 0 scans every forward arc, 465 of them for 62 vertices, and the
    reference pops nothing; the host build agrees (the CUDA build is checked in test_repeat_graphs_gpu.py)."""
    g, prm = fuzz_graph(ref, "dense31")
    arcs, seq, _, _, _ = ref.read_graph(g)
    assert len(arcs) == 930 and len(arcs) // 2 > 4 * 2 * len(seq)
    assert FixStepper(ref, sim).step("asg_pop_bubble", g, prm["bub_dist"]) == 0
    ref.asg_destroy(g)


# ---- what each set is for ----------------------------------------------------------------------------------------------

EXPECT = {
    "direct_short": {"branching", "links"},
    "direct_long": {"branching", "links", "bubbles"},
    "inverted": {"branching", "links", "bubbles"},
    "tandem": {"branching", "links", "circular", "biloops", "internal"},
    "plasmids": {"branching", "links", "circular"},
    "het30k": {"bubbles", "long_walk"},
}


def _clean_counting(lib, g, o):
    n = Counter()

    def step(fn, g, *args):
        c = getattr(lib, fn)(g, *args)
        n[fn] += c & 0xffffffff
        return c
    step("asg_arc_del_trans", g, o.gap_fuzz)
    clean_passes(step, lib, g, o)
    return n


@pytest.mark.parametrize("name", SETS)
def test_set_reaches_its_topology(name, lpafs, ref, port):
    """On the reference's own result (the port's where the reference is not built; the port equals it step by step above)."""
    lib = ref if ref is not None else port
    r = Pipeline(lib, lpafs[name], opt=layout_paf.opt_for(lib, name)).read().select().sg_gen()
    n = _clean_counting(lib, r.sg, r.opt)
    arcs = lib.read_graph(r.sg)[0]
    live = arcs[(arcs["ol_del"] & DEL) == 0]
    deg = np.bincount((live["ul"] >> np.uint64(32)).astype(np.int64))
    gfa = r.ug_gen().gfa().decode().splitlines()
    seen = set()
    if (deg >= 2).any():
        seen.add("branching")
    if any(ln.startswith("L\t") for ln in gfa):
        seen.add("links")
    if any(ln.startswith("S\t") and ln.split("\t")[1].endswith("c") for ln in gfa):
        seen.add("circular")
    if n["asg_pop_bubble"]:
        seen.add("bubbles")
    if n["asg_cut_biloop"]:
        seen.add("biloops")
    if n["asg_cut_internal"]:
        seen.add("internal")
    r.free()
    if name == "het30k":
        # the reads inside the heterozygous region that are still in the graph when bubbles are first popped: the walk from the
        # region's source visits all of them, more than the CUDA build's initial scratch of 64 vertices
        r = Pipeline(lib, lpafs[name], opt=layout_paf.opt_for(lib, name)).read().select().sg_gen()
        lib.asg_arc_del_trans(r.sg, r.opt.gap_fuzz)
        lib.asg_cut_tip(r.sg, r.opt.max_ext)
        names, (arcs, seq) = r.names(), lib.read_graph(r.sg)[:2]
        het = layout_paf.het_reads(name)
        has_arc = set((arcs["ul"] >> np.uint64(33)).tolist())
        n_het = sum(1 for i, nm in enumerate(names) if nm.decode() in het and not seq[i] & DEL and i in has_arc)
        print(name, "reads of the heterozygous region in the graph:", n_het)
        if n_het > 64:
            seen.add("long_walk")
        r.free()
    print(name, dict(n), sorted(seen))
    assert EXPECT[name] <= seen, EXPECT[name] - seen
