"""CPU tier: the oracle port step by step against the unmodified reference (oracle/_ref/libminiasm_ref.so) --
this is what pins the restatement, since the reference has no tests of its own.  The reference's results are stored
digests (tests/refgold.py); each step starts from the port's own pre-state."""
import ctypes as C
import numpy as np
import pytest

from miniasm_b200 import capi, synth
from oracle import loaders
from miniasm_b200.pipeline import Pipeline, canon_arcs

SETS = ["tiny_exact", "chaos_small", "chaos", "bubbles800", "shuffled", "lowcov", "varlen300", "skew_small", "c1_ecoli_like"]


@pytest.fixture(scope="module")
def port(built):
    return loaders.load_oracle_port()


def mask(h):
    h = h.copy()
    h["bl_del"] &= 0x7fffffff
    return h


def _graph(lib, g):
    a, s, i, srt, symm = lib.read_graph(g)
    return [a, s, i, srt, symm]


@pytest.mark.parametrize("name", SETS)
def test_port_matches_reference_stepwise(name, ref, port, paf_dir, gold):
    paf = synth.generate(name, f"{paf_dir}/{name}.paf")
    hits = lambda q: [q.names(), np.sort(mask(q.hits_np()), order=list(capi.HIT_DT.names))]
    p = Pipeline(port, paf).read()

    def read_ref():
        r = Pipeline(ref, paf).read()
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
    o = p.opt

    def run(lib, fn, args):
        arcs, seq, idx, srt, symm = port.read_graph(p.sg)
        g2 = lib.make_graph(arcs, seq, srt, symm)
        if idx is not None:
            g2.contents.idx = capi.c_malloc_copy(idx)
        n = getattr(lib, fn)(g2, *args)
        out = [n] + _graph(lib, g2)
        lib.asg_destroy(g2)
        return out
    for fn, args in [("asg_arc_del_trans", (o.gap_fuzz,)), ("asg_cut_tip", (o.max_ext,)), ("asg_pop_bubble", (o.bub_dist,)),
                     ("asg_arc_del_short", (0.5,)), ("asg_cut_tip", (o.max_ext,)), ("asg_pop_bubble", (o.bub_dist,)),
                     ("asg_arc_del_short", (0.7,)), ("asg_cut_internal", (1,)), ("asg_cut_biloop", (o.max_ext,)),
                     ("asg_cut_tip", (o.max_ext,)), ("asg_pop_bubble", (o.bub_dist,)), ("asg_arc_del_short", (0.8,))]:
        gold.expect(run(port, fn, args), lambda: run(ref, fn, args))     # same pre-state for both
        getattr(port, fn)(p.sg, *args)

    def unitigs(lib):
        ug = lib.ma_ug_gen(p.sg)
        text = lib.print_to_string("ma_ug_print", ug, p.d, p.sub)
        lib.ma_ug_destroy(ug)
        return text
    gold.expect(unitigs(port), lambda: unitigs(ref))
    p.free()


def test_tie_order_audit(ref, port, paf_dir, gold):
    """SURVEY.md section 7.1: the reference's radix sort is unstable, ours (port and CUDA) are stable.  On data with
    thousands of tied sort keys the final GFA must not depend on it."""
    for name in ("jitter30", "chaos"):
        paf = synth.generate(name, f"{paf_dir}/{name}.paf")
        gold.expect(Pipeline(port, paf).run_all(), lambda: Pipeline(ref, paf).run_all())


def _reduce_tied(lib, w2_first):
    from tests.tied_graph import FUZZ, tied_graph
    arcs, seq, idx = tied_graph(w2_first)
    g = lib.make_graph(arcs, seq, is_srt=True)
    g.contents.idx = capi.c_malloc_copy(idx)
    n = lib.asg_arc_del_trans(g, FUZZ)
    out = lib.read_graph(g)
    lib.asg_destroy(g)
    return n, out


def test_tied_arcs_decide_the_counter_not_the_graph(ref, port, gold):
    """ADVICE round 1: two arcs tied on (source, length) whose targets overlap each other.  Which one the reference explores first
    changes how many arcs asg_arc_del_trans itself reduces (asg.c:164-171); asg_symm inside the call (asg.c:188-191) takes the
    one-sided survivor, so the graph that comes out is the same.  The port follows the reference for either slab order."""
    res = {}
    for w2_first in (False, True):
        n_p, gp = _reduce_tied(port, w2_first)
        gold.expect([n_p, *gp], lambda: (lambda n, g: [n, *g])(*_reduce_tied(ref, w2_first)))
        res[w2_first] = (n_p, gp)
    assert res[True][0] == res[False][0] + 1                     # v -> x is reduced by the pass itself only when w2 comes first
    assert np.array_equal(canon_arcs(res[True][1][0]), canon_arcs(res[False][1][0]))
    assert len(res[True][1][0]) == 6                             # v -> w1 -> w2 -> x and the complement chain remain


@pytest.mark.parametrize("args", ["-n 4000 -l 2000 -L 30000 -c 30 -j 100 -s 41", "-n 6000 -l 1500 -L 40000 -c 40 -j 300 -s 42 -d 20000"])
@pytest.mark.parametrize("hang,frac", [(1000, 0.8), (200, 0.5), (4000, 0.95)])
def test_port_no_cont(args, hang, frac, ref, port, paf_dir, gold):
    """-R (SURVEY.md 8f row 2): ma_hit_no_cont (hit.c:38-68) and ma_hit_read with its exclusion list (hit.c:86) -- read lengths
    spread over a factor of 20, so many reads lie clearly inside a read twice as long."""
    paf = synth.generate(args, f"{paf_dir}/nocont_{len(args)}.paf").encode()
    names = lambda d: [(d.contents.seq[i].name, d.contents.seq[i].len) for i in range(d.contents.n_seq)]

    def no_cont(lib):
        excl = lib.ma_hit_no_cont(paf, 2000, 100, hang, frac)
        d, n = lib.sd_init(), C.c_size_t(0)
        h = lib.ma_hit_read(paf, 2000, 100, d, C.byref(n), 1, excl)
        a = mask(capi.np_from_ptr(h, n.value, capi.HIT_DT))
        out = [names(excl), names(d), np.sort(a, order=list(capi.HIT_DT.names))]
        capi.c_free(h), lib.sd_destroy(d), lib.sd_destroy(excl)
        return out
    got = no_cont(port)
    gold.expect(got, lambda: no_cont(ref))
    assert len(got[0]) > 20 or hang == 4000
    gone = {nm for nm, _ in got[0]}
    assert gone and not gone & {nm for nm, _ in got[1]}


@pytest.mark.parametrize("style,ext", [("fa_wrap", "fa"), ("fa_one_crlf", "fa"), ("fa_var_gaps_extra_dups_missing", "fa"), ("fa_wrap", "fa.gz"),
                                       ("fq", "fq"), ("fq_crlf_extra_dups", "fq"), ("fq_missing", "fq.gz"), ("fq_multi", "fq")])
def test_port_ug_seq(style, ext, ref, port, paf_dir, gold):
    """-f reads (SURVEY.md 8f row 3): ma_ug_seq (asm.c:236-290 over kseq.h:163-211) -- FASTA / FASTQ, wrapped, CRLF, gzip, empty
    lines, multi-line FASTQ, records missing / foreign / repeated; the port fills the unitigs the port built, the reference the ones
    it built."""
    from tests.test_cli_gpu import _reads_file
    paf = synth.generate("chaos_small", f"{paf_dir}/chaos_small.paf")
    reads = _reads_file(paf, f"{paf_dir}/port_{style}.{ext}", style).encode()
    got = Pipeline(port, paf).run_all(reads.decode())
    gold.expect(got, lambda: Pipeline(ref, paf).run_all(reads.decode()))
    assert b"\t*\tLN" not in got and got.count(b"S\t") > 0
    r = Pipeline(port, paf).read().select().sg_gen().clean()
    assert port.ma_ug_seq(port.ma_ug_gen(r.sg), r.d, r.sub, b"/nonexistent/reads.fa") == -1      # asm.c:243
    r.free()
