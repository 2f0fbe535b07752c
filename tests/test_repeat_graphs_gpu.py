"""GPU parity of stage (iii) -- the cleaning passes, the unitigs and the GFA -- on layouts with repeats, inverted repeats,
tandem arrays, plasmids and a heterozygous region (tests/layout_paf.py) and on motif graphs (tests/graph_fuzz.py), against
the unmodified reference: pass by pass through the drop-in ABI, through the command line and through the fused path.  The
reference's results are stored digests (tests/refgold.py)."""
import ctypes as C
import os
import subprocess
import sys

import pytest

from miniasm_b200 import capi
from miniasm_b200.pipeline import Pipeline
from tests import graph_fuzz, layout_paf
from tests.refgold import RECORD
from tests.test_asg_gpu import _cleanup, _cleanup_symm, _run
from tests.test_clean_gpu import Stepper, _unitigs
from tests.test_cli_gpu import OURS, REF, _counters, run, same
from tests.test_repeat_graphs_cpu import clean_passes, fuzz_graph

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SETS = list(layout_paf.SETS)
FUZZ = list(graph_fuzz.CASES)


@pytest.fixture(scope="module")
def lpafs(built, paf_dir):
    out = {name: layout_paf.generate(name, f"{paf_dir}/lp_{name}.paf") for name in SETS}
    for name, path in out.items():
        assert layout_paf.sha256(path) == layout_paf.SHA256[name], name      # the stored digests are of these bytes
    return out


def _args(name, path, *opts):
    return layout_paf.CLI_OPTS.get(name, []) + list(opts) + [path]


# ---- the drop-in ABI, pass by pass ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", SETS)
def test_cleaning_passes_stepwise(name, lpafs, port, ref, prod, gold):
    r = Pipeline(port, lpafs[name], opt=layout_paf.opt_for(port, name)).read().select().sg_gen()
    step = Stepper(port, ref, prod, gold)
    step("asg_arc_del_trans", r.sg, r.opt.gap_fuzz)
    clean_passes(step, port, r.sg, r.opt)
    tp, tq = _unitigs(prod, port, r.sg, r), _unitigs(prod, prod, r.sg, r)
    want = lambda: _unitigs(ref, ref, r.sg, r)
    gold.expect(tp, want)
    gold.expect(tq, want)
    r.free()


@pytest.mark.parametrize("name", FUZZ)
def test_cleaning_passes_on_motif_graphs(name, port, ref, prod, gold):
    """Each pass alone on the raw motif graph, then the whole stage (iii) from asg_arc_del_trans on."""
    g, prm = fuzz_graph(port, name)
    o = port.default_opt()
    step = Stepper(port, ref, prod, gold)
    for fn, arg in (("asg_pop_bubble", prm["bub_dist"]), ("asg_cut_tip", prm["max_ext"]), ("asg_cut_internal", 1),
                    ("asg_cut_biloop", prm["max_ext"]), ("asg_cut_internal", prm["max_ext"])):
        h = port.clone_graph(g)
        step(fn, h, arg)
        port.asg_destroy(h)
    step("asg_arc_del_trans", g, o.gap_fuzz)
    clean_passes(step, port, g, o, prm["max_ext"], prm["bub_dist"])
    port.asg_destroy(g)


@pytest.mark.parametrize("name", FUZZ)
def test_cleanup_and_symm_on_motif_graphs(name, port, ref, prod, gold):
    """asg_cleanup and asg_cleanup + asg_symm on the motif graph's arcs in random order (test_asg_gpu.py's comparisons)."""
    arcs, seq, _ = graph_fuzz.build(name)
    g = port.make_graph(arcs, seq)
    gold.expect(_run(prod, port, g, _cleanup, exact_order=False), lambda: _run(ref, port, g, _cleanup, exact_order=False))
    gold.expect(_run(prod, port, g, _cleanup_symm, exact_order=False), lambda: _run(ref, port, g, _cleanup_symm, exact_order=False))
    port.asg_destroy(g)


DENSE = r'''
import sys
sys.path.insert(0, sys.argv[1])
from miniasm_b200 import capi
from tests import graph_fuzz
lib = capi.load_product()
lib.set_verbose(0)
arcs, seq, prm = graph_fuzz.build("dense31")
g = lib.make_graph(arcs, seq)
lib.asg_cleanup(g)
print(lib.asg_pop_bubble(g, prm["bub_dist"]))
'''


@pytest.mark.skipif(RECORD, reason="runs the CUDA library only")
def test_dense_graph_bubble_walk_fits_its_scratch(built):
    """The dense motif graph (31 reads, all 465 pairs overlapping, not transitively reduced): the walk from read 0 scans 465
    arcs, more than 4 per vertex.  The scratch must grow to what the walk needs and the call return the reference's count
    (0, tests/test_repeat_graphs_cpu.py); it runs in its own process so that an exit of the library is a failure here."""
    r = subprocess.run([sys.executable, "-c", DENSE, ROOT], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split() == ["0"]


# ---- the command line ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", SETS)
def test_default_gfa_and_counters(name, lpafs, gold):
    args = _args(name, lpafs[name])
    out = same(gold, args)
    assert out.startswith(b"S\tutg000001")
    gold.cli("counters", args, _counters(run(OURS, args)[2]), lambda: _counters(run(REF, args)[2]))


@pytest.mark.parametrize("stage", [6, 7, 9, 10])
@pytest.mark.parametrize("name", ["inverted", "tandem", "plasmids", "het30k"])
def test_stage_dumps(name, stage, lpafs, gold):
    same(gold, _args(name, lpafs[name], "-S", str(stage), "-p", "ug"))
    same(gold, _args(name, lpafs[name], "-S", str(stage), "-p", "sg"), exact=False)


@pytest.mark.parametrize("name", ["tandem", "plasmids"])
def test_gfa_with_reads(name, lpafs, paf_dir, gold):
    reads = os.path.join(paf_dir, f"lp_{name}.fa")
    with open(reads, "w") as f:
        f.write(layout_paf.layout(name).reads_fasta())
    out = same(gold, _args(name, lpafs[name], "-f", reads))
    assert b"\tLN:i:" in out and b"\t*\tLN" not in out


@pytest.mark.parametrize("name", SETS)
def test_no_containment_filter(name, lpafs, gold):
    same(gold, _args(name, lpafs[name], "-R"))


# ---- the fused path --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", SETS)
def test_fused_path_gfa(name, lpafs, prod, gold):
    """mab_load_ingest_text -> mab_select -> mab_layout -> mab_unitigs -> mab_write_gfa prints the reference's GFA."""
    paf = lpafs[name]
    args = _args(name, paf)
    want = lambda: subprocess.run([REF] + args, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout
    got = None
    if not RECORD:
        data = open(paf, "rb").read()
        opt = layout_paf.opt_for(prod, name)
        ctx = prod.mab_create(0)
        assert prod.mab_load_ingest_text(ctx, data, len(data), opt.min_span, opt.min_match, 1) == 0
        prod.mab_select(ctx, C.byref(opt), 0, 0, 100)
        prod.mab_layout(ctx, C.byref(opt), 100)
        prod.mab_unitigs(ctx)
        out = os.path.join(os.path.dirname(paf), f"fused_{name}.gfa")
        fp = capi._libc.fopen(out.encode(), b"w")
        prod.mab_write_gfa(ctx, fp)
        capi._libc.fclose(fp)
        prod.mab_destroy(ctx)
        got = open(out, "rb").read()
    gold.cli("GFA", args, got, want)


def test_one_rank_sharded_run(lpafs, paf_dir, gold):
    """The sharded pipeline (tests/shard_worker.py) with one rank on the tandem set."""
    paf = lpafs["tandem"]
    out = os.path.join(paf_dir, "lp_tandem_shard1.gfa")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=1", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tests", "shard_worker.py"), paf, out]
    want = lambda: subprocess.run([REF, paf], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout
    if not RECORD:
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-3000:]
    gold.cli("GFA", [paf], None if RECORD else open(out, "rb").read(), want)
