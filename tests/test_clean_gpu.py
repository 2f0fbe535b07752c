"""GPU parity of stage (iii) (SURVEY.md 8a rows a18-a25): the order-dependent cleaning passes, unitig
construction and the final GFA, against the unmodified reference on graphs with tips, bubbles, short
overlaps, internal sequences and bi-loops.  Pre-states come from the oracle port; the reference's results for them are stored
digests (tests/refgold.py)."""
import ctypes as C
import gzip
import os

import numpy as np
import pytest

from miniasm_b200 import capi, synth
from miniasm_b200.pipeline import Pipeline, gfa_canon

pytestmark = pytest.mark.gpu

NOISY = ["bubbles800", "chaos", "chaos_small", "shuffled", "varlen300", "lowcov", "c1_ecoli_like", "jitter30"]
ALL = NOISY + ["tiny_exact", "small_exact", "skew_small"]


@pytest.fixture(scope="module")
def pafs(paf_dir):
    return {name: synth.generate(name, f"{paf_dir}/{name}.paf") for name in ALL}


def _clone_to(lib, src_lib, g):
    arcs, seq, idx, srt, symm = src_lib.read_graph(g)
    h = lib.make_graph(arcs, seq, srt, symm)
    if idx is not None:
        h.contents.idx = capi.c_malloc_copy(idx)
    return h


def _state(lib, g):
    a, s, i, f1, f2 = lib.read_graph(g)
    return [a, s, f1, f2, i]


class Stepper:
    """Runs the passes on a graph the oracle port owns: each pass runs on a clone of the current pre-state in the library under
    test and is compared (count and graph) with what the reference gives from that pre-state; the port then advances the graph."""

    def __init__(self, port, ref, prod, gold):
        self.port, self.ref, self.prod, self.gold = port, ref, prod, gold

    def _on(self, lib, name, g, args):
        h = _clone_to(lib, self.port, g)
        n = getattr(lib, name)(h, *args)
        out = (n, _state(lib, h))
        lib.asg_destroy(h)
        return out

    def __call__(self, name, g, *args):
        self.gold.expect(self._on(self.prod, name, g, args), lambda: self._on(self.ref, name, g, args))
        return getattr(self.port, name)(g, *args)


def _unitigs(lib, writer, g, r):
    """ma_ug_gen of lib on a clone of g, printed by writer's ma_ug_print."""
    h = _clone_to(lib, r.lib, g)
    ug = lib.ma_ug_gen(h)
    text = writer.print_to_string("ma_ug_print", ug, r.d, r.sub)
    lib.ma_ug_destroy(ug), lib.asg_destroy(h)
    return text


@pytest.mark.parametrize("name", NOISY)
def test_cleaning_passes_stepwise(name, pafs, port, ref, prod, gold):
    r = Pipeline(port, pafs[name]).read().select().sg_gen()
    o, g = r.opt, r.sg
    step = Stepper(port, ref, prod, gold)
    port.asg_arc_del_trans(g, o.gap_fuzz)
    step("asg_cut_tip", g, o.max_ext)
    step("asg_pop_bubble", g, o.bub_dist)
    for i in range(o.n_rounds + 1):
        ratio = float(np.float32(o.min_ovlp_drop_ratio) + (np.float32(o.max_ovlp_drop_ratio) - np.float32(o.min_ovlp_drop_ratio))
                      / np.float32(o.n_rounds) * np.float32(i))
        if step("asg_arc_del_short", g, ratio):
            step("asg_cut_tip", g, o.max_ext)
            step("asg_pop_bubble", g, o.bub_dist)
    step("asg_cut_internal", g, 1)
    step("asg_cut_biloop", g, o.max_ext)
    step("asg_cut_tip", g, o.max_ext)
    step("asg_pop_bubble", g, o.bub_dist)
    if step("asg_arc_del_short", g, o.final_ovlp_drop_ratio):
        step("asg_cut_tip", g, o.max_ext)
        step("asg_pop_bubble", g, o.bub_dist)
    # unitigs from the cleaned graph: the product's structs through the port's writer and through ours
    tp, tq = _unitigs(prod, port, g, r), _unitigs(prod, prod, g, r)
    want = lambda: _unitigs(ref, ref, g, r)
    gold.expect(tp, want)
    gold.expect(tq, want)
    r.free()


@pytest.mark.parametrize("ext,dist", [(1, 50000), (2, 5000), (8, 200000), (20, 1000)])
def test_cleaning_other_parameters(ext, dist, pafs, port, ref, prod, gold):
    r = Pipeline(port, pafs["chaos"]).read().select().sg_gen()
    g = r.sg
    step = Stepper(port, ref, prod, gold)
    port.asg_arc_del_trans(g, 1000)
    step("asg_cut_tip", g, ext)
    step("asg_pop_bubble", g, dist)
    step("asg_cut_internal", g, ext)
    step("asg_cut_biloop", g, ext)
    r.free()


@pytest.mark.parametrize("name", ["chaos", "bubbles800", "tiny_exact"])
def test_ug_gen_on_raw_graph(name, pafs, port, ref, prod, gold):
    """`-S5 -p ug`: unitigs straight from ma_sg_gen's graph (not symmetric: the literal replay path)."""
    r = Pipeline(port, pafs[name]).read().select().sg_gen()
    gold.expect(_unitigs(prod, port, r.sg, r), lambda: _unitigs(ref, ref, r.sg, r))
    r.free()


@pytest.mark.parametrize("name", ALL)
def test_gfa_end_to_end(name, pafs, ref, prod, gold):
    """The whole drop-in path, every call on the GPU: byte-identical GFA (and equal as sorted S/L/a/x multisets)."""
    tp = Pipeline(prod, pafs[name]).run_all()
    gold.expect(gfa_canon(tp), lambda: gfa_canon(Pipeline(ref, pafs[name]).run_all()))
    gold.expect(tp, lambda: Pipeline(ref, pafs[name]).run_all())


def _write_reads(paf, path, gz=False, fastq=False):
    lens = {}
    with open(paf) as f:
        for line in f:
            t = line.split("\t")
            lens[t[0]] = int(t[1]); lens[t[5]] = int(t[6])
    rng = np.random.default_rng(3)
    op = gzip.open if gz else open
    with op(path, "wt") as f:
        for k, (nm, ln) in enumerate(sorted(lens.items())):
            s = "".join(np.array(list("ACGTNacgtRY"))[rng.integers(0, 11, ln)])
            if fastq:
                f.write(f"@{nm} extra comment\n{s}\n+\n{'I' * ln}\n")
            else:
                f.write(f">{nm}\n" + "\n".join(s[i:i + 70] for i in range(0, ln, 70)) + "\n")
    return path


@pytest.mark.parametrize("fmt", ["fa", "fq.gz"])
def test_gfa_with_sequences(fmt, pafs, ref, prod, paf_dir, gold):
    """-f reads: S lines carry the unitig sequence (ma_ug_seq, asm.c:236-290)."""
    paf = pafs["chaos_small"]
    reads = _write_reads(paf, os.path.join(paf_dir, f"reads.{fmt}"), gz=fmt.endswith("gz"), fastq=fmt.startswith("fq"))
    tp = Pipeline(prod, paf).run_all(reads)
    gold.expect(tp, lambda: Pipeline(ref, paf).run_all(reads))
    assert b"\tLN:i:" in tp and not tp.startswith(b"S\tutg000001l\t*")
