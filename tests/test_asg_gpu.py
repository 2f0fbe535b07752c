"""GPU parity of the string-graph container passes (SURVEY.md 8a rows a12-a18) against the
unmodified reference, function by function through the C ABI, on graphs the oracle port built (the reference's results
for the same pre-states are stored digests, tests/refgold.py)."""
import ctypes as C

import numpy as np
import pytest

from miniasm_b200 import capi, synth
from miniasm_b200.capi import ARC_DT, DEL
from miniasm_b200.pipeline import Pipeline, canon_arcs
from tests.tied_graph import FUZZ, tied_graph

pytestmark = pytest.mark.gpu

SETS = ["tiny_exact", "small_exact", "jitter30", "varlen300", "bubbles800", "chaos", "skew_small", "lowcov"]


@pytest.fixture(scope="module")
def graphs(port, paf_dir):
    """name -> port pipeline stopped right after ma_sg_gen (sorted + indexed raw graph)."""
    out = {}
    for name in SETS:
        paf = synth.generate(name, f"{paf_dir}/{name}.paf")
        out[name] = Pipeline(port, paf).read().select().sg_gen()
    yield out
    for p in out.values():
        p.free()


def _clone_to(lib, src_lib, g):
    arcs, seq, idx, srt, symm = src_lib.read_graph(g)
    h = lib.make_graph(arcs, seq, srt, symm)
    if idx is not None:
        h.contents.idx = capi.c_malloc_copy(idx)
    return h


def _state(lib, g, exact_order=True):
    """What the comparison of two graphs looks at; with exact_order=False the arcs are compared by their sort keys position by
    position and as a canonical multiset (the reference's radix sort is unstable: ties may permute)."""
    a, s, i, srt, symm = lib.read_graph(g)
    arcs = [a] if exact_order else [a["ul"], canon_arcs(a)]
    return [len(a), s, srt, symm, *arcs, i]


def _run(lib, src_lib, g, fn, *args, exact_order=True):
    """fn(lib, clone of g) -> (its return value, state of the clone afterwards)."""
    h = _clone_to(lib, src_lib, g)
    n = fn(lib, h, *args)
    out = (n, _state(lib, h, exact_order))
    lib.asg_destroy(h)
    return out


def _del_trans(lib, g, fuzz):
    return lib.asg_arc_del_trans(g, fuzz)


@pytest.mark.parametrize("name", SETS)
def test_del_trans(name, graphs, port, ref, prod, gold):
    p = graphs[name]
    gold.expect(_run(prod, port, p.sg, _del_trans, p.opt.gap_fuzz), lambda: _run(ref, port, p.sg, _del_trans, p.opt.gap_fuzz))


@pytest.mark.parametrize("fuzz", [0, 10, 100000])
def test_del_trans_fuzz(fuzz, graphs, port, ref, prod, gold):
    p = graphs["chaos"]
    gold.expect(_run(prod, port, p.sg, _del_trans, fuzz), lambda: _run(ref, port, p.sg, _del_trans, fuzz))


def _graph_with_idx(lib, arcs, seq, idx):
    g = lib.make_graph(arcs, seq, True)
    g.contents.idx = capi.c_malloc_copy(idx)
    return g


def test_del_trans_deleted_reads(graphs, port, ref, prod, gold):
    """reads flagged del lose every arc (asg.c:158-161)."""
    p = graphs["jitter30"]
    arcs, seq, idx, _, _ = port.read_graph(p.sg)
    seq = seq.copy()
    seq[::7] |= DEL
    g = _graph_with_idx(port, arcs, seq, idx)
    gold.expect(_run(prod, port, g, _del_trans, 1000), lambda: _run(ref, port, g, _del_trans, 1000))
    port.asg_destroy(g)


@pytest.mark.parametrize("w2_first", [False, True])
def test_del_trans_tied_arcs(w2_first, port, ref, prod, gold):
    """Two arcs tied on (source, length) whose targets overlap each other (tests/tied_graph.py): for either slab order the kernel
    reduces what the reference's sequential walk reduces -- the counter differs between the two orders, never between the two sides."""
    g = _graph_with_idx(port, *tied_graph(w2_first))
    got = _run(prod, port, g, _del_trans, FUZZ)
    assert got[0] == (4 if w2_first else 3)                    # v -> x is reduced by the pass itself only when w2 is walked first
    gold.expect(got, lambda: _run(ref, port, g, _del_trans, FUZZ))
    port.asg_destroy(g)


def _cleanup(lib, g):
    lib.asg_cleanup(g)


@pytest.mark.parametrize("name", ["small_exact", "chaos", "skew_small"])
def test_cleanup_sorts_and_indexes(name, graphs, port, ref, prod, gold):
    """asg_cleanup on a shuffled, partly deleted arc set: rm + sort + index (asg.c:57-80)."""
    p = graphs[name]
    arcs, seq, _, _, _ = port.read_graph(p.sg)
    rng = np.random.default_rng(7)
    arcs = arcs[rng.permutation(len(arcs))].copy()
    arcs["ol_del"][rng.random(len(arcs)) < 0.1] |= DEL
    seq = seq.copy()
    seq[rng.random(len(seq)) < 0.02] |= DEL
    g = port.make_graph(arcs, seq)
    got = _run(prod, port, g, _cleanup, exact_order=False)   # the reference's radix sort is unstable: ties may permute
    gold.expect(got, lambda: _run(ref, port, g, _cleanup, exact_order=False))
    ul = got[1][4]
    assert np.all(ul[1:] >= ul[:-1])
    port.asg_destroy(g)


def _cleanup_symm(lib, g):
    lib.asg_cleanup(g)
    lib.asg_symm(g)


@pytest.mark.parametrize("name", ["chaos", "bubbles800", "skew_small"])
def test_symm(name, graphs, port, ref, prod, gold):
    """asg_symm = del_multi + del_asymm (asg.c:104-145) on a graph with planted duplicates / one-sided arcs."""
    p = graphs[name]
    arcs, seq, _, _, _ = port.read_graph(p.sg)
    rng = np.random.default_rng(11)
    dup = arcs[rng.random(len(arcs)) < 0.01].copy()
    dup["ul"] += 3                                          # same source + target, longer: a multi-arc
    arcs = np.concatenate([arcs[rng.random(len(arcs)) > 0.01], dup])
    g = port.make_graph(arcs, seq)
    gold.expect(_run(prod, port, g, _cleanup_symm, exact_order=False), lambda: _run(ref, port, g, _cleanup_symm, exact_order=False))
    port.asg_destroy(g)


def _del_short(lib, g, ratio):
    return lib.asg_arc_del_short(g, ratio)


@pytest.mark.parametrize("ratio", [0.5, 0.6, 0.7, 0.8, 0.95])
def test_del_short(ratio, graphs, port, ref, prod, gold):
    p = graphs["chaos"]
    g = port.clone_graph(p.sg)
    port.asg_arc_del_trans(g, 1000)
    gold.expect(_run(prod, port, g, _del_short, ratio), lambda: _run(ref, port, g, _del_short, ratio))
    port.asg_destroy(g)


def test_big_slabs(port, ref, prod, gold):
    """A hub vertex beyond the warp kernel (128 arcs) and beyond the CTA kernel (8192 arcs)."""
    rng = np.random.default_rng(5)
    n_seq = 12000
    seq = np.full(n_seq, 20000, dtype=np.uint32)
    rows = []
    def add(u, v, l):
        rows.append((u << 32 | l, v, 20000 - l))
        rows.append(((v ^ 1) << 32 | l, u ^ 1, 20000 - l))
    for hub, deg in ((0, 300), (2, 5000), (4, 9000)):
        tg = rng.choice(np.arange(6, 2 * n_seq), size=deg, replace=False)
        ls = np.sort(rng.integers(1, 18000, size=deg))
        for t, l in zip(tg, ls):
            add(hub, int(t), int(l))
        for k in range(0, deg - 1, 3):                      # chain some targets so that reductions happen
            add(int(tg[k]), int(tg[k + 1]), int(max(1, ls[k + 1] - ls[k])))
    arcs = np.array(rows, dtype=ARC_DT)
    g = port.make_graph(arcs, seq)
    port.asg_cleanup(g)                # same slab order on both sides: lengths tie heavily here (DESIGN.md "tie order")
    gold.expect(_run(prod, port, g, _del_trans, 1000), lambda: _run(ref, port, g, _del_trans, 1000))
    port.asg_destroy(g)


def test_empty_graph(prod):
    seq = np.full(10, 5000, dtype=np.uint32)
    gp = prod.make_graph(np.zeros(0, dtype=ARC_DT), seq)
    prod.asg_cleanup(gp)
    assert prod.asg_arc_del_trans(gp, 1000) == 0
    arcs, s, idx, srt, _ = prod.read_graph(gp)
    assert len(arcs) == 0 and srt and idx is not None and not idx.any()
    prod.asg_destroy(gp)
