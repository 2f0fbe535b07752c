"""mab_write_paf / mab_write_bed / mab_write_sg (dump_dev.cu): the -p paf|bed|sg texts formatted on the GPU and written in chunks.
Each must give exactly the bytes of the export route on the same context: print_hits / print_subs restated in Python over
mab_export_hits/_dict/_sub, and the library's ma_sg_print over mab_export_sg/_dict/_sub.  Config 2 spans many windows and chunks
of the writer; its command lines are also held to the reference's digests (tests/golden/dump_writers_digests.json)."""
import ctypes as C
import json
import os

import pytest

from miniasm_b200 import capi, synth
from miniasm_b200.capi import HIT_DT, SUB_DT
from tests import refgold
from tests.test_cli_gpu import OURS, REF, outcome, run
from tests.test_dump_writers_cpu import py_bed, py_paf

pytestmark = pytest.mark.gpu

DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dump_writers_digests.json")

SETS = ["chaos_small", "chaos", "bubbles800", "tiny_exact", "shuffled", "skew_small"]
SELECTIONS = {"S2": dict(stage=2), "S3": dict(stage=3), "S4": dict(stage=4), "S5": dict(stage=5), "default": dict(),
              "no1": dict(no_first=1), "no2": dict(no_second=1), "no1no2": dict(no_first=1, no_second=1),
              "R": dict(nocont=True), "b": dict(bi_dir=0)}


@pytest.fixture(scope="module")
def pafs(built, paf_dir):
    return {name: synth.generate(name, f"{paf_dir}/{name}.paf") for name in SETS}


def selected(prod, paf, no_first=0, no_second=0, stage=100, nocont=False, bi_dir=1):
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    assert prod.mab_load_paf_file(ctx, paf.encode()) == 0
    if nocont:
        prod.mab_ingest_nocont(ctx, opt.min_span, opt.min_match, bi_dir, opt.max_hang, opt.int_frac)
    else:
        prod.mab_ingest(ctx, opt.min_span, opt.min_match, bi_dir)
    prod.mab_select(ctx, C.byref(opt), no_first, no_second, stage)
    return ctx, opt


def written(fn, ctx, path):
    """(return value, bytes in the file) of a writer called on a FILE opened for `path`"""
    fp = capi._libc.fopen(path.encode(), b"w")
    n = fn(ctx, fp)
    capi._libc.fclose(fp)
    with open(path, "rb") as f:
        return n, f.read()


def exported(prod, ctx):
    d = prod.mab_export_dict(ctx)
    names = [d.contents.seq[i].name for i in range(d.contents.n_seq)]
    sp = prod.mab_export_sub(ctx)
    sub = capi.np_from_ptr(sp, len(names), SUB_DT) if sp else None
    n = C.c_size_t(0)
    hp = prod.mab_export_hits(ctx, C.byref(n))
    hits = capi.np_from_ptr(hp, n.value, HIT_DT)
    capi.c_free(hp), capi.c_free(sp), prod.sd_destroy(d)
    return names, sub, hits


def check_paf_bed(prod, ctx, tmp_path):
    n_paf, paf = written(prod.mab_write_paf, ctx, str(tmp_path / "o.paf"))
    n_bed, bed = written(prod.mab_write_bed, ctx, str(tmp_path / "o.bed"))
    names, sub, hits = exported(prod, ctx)
    if sub is None:                                   # -1 -2: no interval table, nothing to print
        assert (n_paf, paf, n_bed, bed) == (-1, b"", -1, b"")
        return paf, bed
    assert paf == py_paf(hits, names, sub) and n_paf == len(paf)
    assert bed == py_bed(names, sub) and n_bed == len(bed)
    return paf, bed


def check_sg(prod, ctx, tmp_path):
    n, got = written(prod.mab_write_sg, ctx, str(tmp_path / "o.sg"))
    g, d, sp = prod.mab_export_sg(ctx), prod.mab_export_dict(ctx), prod.mab_export_sub(ctx)
    want = prod.print_to_string("ma_sg_print", g, d, sp)
    prod.asg_destroy(g), prod.sd_destroy(d), capi.c_free(sp)
    assert got == want and n == len(got)
    return got


@pytest.mark.parametrize("sel", list(SELECTIONS))
@pytest.mark.parametrize("name", SETS)
def test_paf_and_bed_match_the_export_route(name, sel, pafs, prod, tmp_path):
    ctx, _ = selected(prod, pafs[name], **SELECTIONS[sel])
    check_paf_bed(prod, ctx, tmp_path)
    prod.mab_destroy(ctx)


@pytest.mark.parametrize("stage", [1, 5, 6, 7, 9, 10, 11])
@pytest.mark.parametrize("name", SETS)
def test_sg_matches_ma_sg_print(name, stage, pafs, prod, tmp_path):
    ctx, opt = selected(prod, pafs[name], stage=stage)
    assert written(prod.mab_write_sg, ctx, str(tmp_path / "none.sg")) == (-1, b"")     # before mab_layout
    prod.mab_layout(ctx, C.byref(opt), stage)
    got = check_sg(prod, ctx, tmp_path)
    assert got.startswith(b"L\t") and (b":" in got.split(b"\t")[1]) == (stage > 1)     # -S 1: no interval table, plain names
    prod.mab_destroy(ctx)


def test_sg_without_read_selection(pafs, prod, tmp_path):
    ctx, opt = selected(prod, pafs["chaos_small"], no_first=1, no_second=1)
    prod.mab_layout(ctx, C.byref(opt), 100)
    got = check_sg(prod, ctx, tmp_path)
    assert got.startswith(b"L\t") and b":" not in got.split(b"\t")[1]
    prod.mab_destroy(ctx)


@pytest.mark.parametrize("content", [b"", b"\n",
                                     b"q\t5000\t0\t4000\t+\tt\t5000\t1000\t5000\t800\t4000\t255\n",    # too shallow for min_dp
                                     b"q\t5000\t0\t100\t+\tt\t5000\t0\t100\t80\t100\t255\n"])          # below min_span
def test_degenerate_inputs_write_nothing(content, prod, tmp_path):
    path = str(tmp_path / "degenerate.paf")
    with open(path, "wb") as f:
        f.write(content)
    for stage in (2, 100):
        ctx, opt = selected(prod, path, stage=stage)
        assert check_paf_bed(prod, ctx, tmp_path) == (b"", b"")
        if stage == 100:
            prod.mab_layout(ctx, C.byref(opt), stage)
            assert check_sg(prod, ctx, tmp_path) == b""
        prod.mab_destroy(ctx)


@pytest.mark.parametrize("name", ["chaos", "skew_small", "bubbles800"])
def test_sharded_context_one_rank(name, pafs, prod, tmp_path):
    """names of a sharded ingest live in the context's name_text"""
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    assert prod.mab_shard_init(ctx, 0, 1, None) == 0
    data = open(pafs[name], "rb").read()
    prod.mab_load_ingest_text_sharded(ctx, data, len(data), opt.min_span, opt.min_match, 1)
    prod.mab_select_sharded(ctx, C.byref(opt))
    prod.mab_layout_sharded(ctx, C.byref(opt))
    got = check_sg(prod, ctx, tmp_path)
    check_paf_bed(prod, ctx, tmp_path)
    prod.mab_destroy(ctx)
    ctx, opt = selected(prod, pafs[name])
    prod.mab_layout(ctx, C.byref(opt), 100)
    assert written(prod.mab_write_sg, ctx, str(tmp_path / "single.sg"))[1] == got
    prod.mab_destroy(ctx)


def test_long_read_names(prod, paf_dir, tmp_path):
    src = synth.generate("tiny_exact", f"{paf_dir}/tiny_exact.paf")
    ren = {"r206": "L" * 70000 + "a", "r27": "L" * 70000 + "b", "r172": "M" * 66000}
    dst = str(tmp_path / "long.paf")
    with open(src) as f, open(dst, "w") as g:
        for line in f:
            c = line.split("\t")
            c[0], c[5] = ren.get(c[0], c[0]), ren.get(c[5], c[5])
            g.write("\t".join(c))
    ctx, opt = selected(prod, dst, stage=2)
    paf, bed = check_paf_bed(prod, ctx, tmp_path)
    assert b"L" * 70000 + b"a\t" in bed and b"M" * 66000 + b"\t" in bed
    prod.mab_destroy(ctx)
    ctx, opt = selected(prod, dst)
    prod.mab_layout(ctx, C.byref(opt), 100)
    check_sg(prod, ctx, tmp_path)
    prod.mab_destroy(ctx)


@pytest.fixture(scope="module")
def c2(built, paf_dir):
    return synth.generate("c2_100k", os.path.join(paf_dir, "c2.paf"))


def test_c2_many_chunks(c2, prod, tmp_path):
    """config 2: ~750 MB of -S 2 paf and ~510 MB of -S 5 sg, i.e. many windows of records and many chunks of text"""
    ctx, opt = selected(prod, c2, stage=2)
    paf, _ = check_paf_bed(prod, ctx, tmp_path)
    assert len(paf) > 500e6
    del paf
    prod.mab_destroy(ctx)
    ctx, opt = selected(prod, c2, stage=5)
    prod.mab_layout(ctx, C.byref(opt), 5)
    assert len(check_sg(prod, ctx, tmp_path)) > 300e6
    prod.mab_destroy(ctx)


@pytest.fixture(scope="module")
def dump_gold():
    """The reference's outcomes of the config-2 command lines, as digests in tests/golden/dump_writers_digests.json, keyed like
    tests/refgold.py keys command lines.  MAB_RECORD_REFERENCE=1 (needs oracle/_ref) records them from the reference binary."""
    table = json.load(open(DIGESTS)) if os.path.exists(DIGESTS) else {}
    recorded = {}

    def check(how, args, got, want):
        key = f"cli {how}: " + " ".join(refgold._file_key(a) if os.path.isfile(a) else a for a in args)
        if refgold.RECORD:
            recorded[key] = refgold.digest(want())
            return
        assert key in table, f"no reference digest for {key}"
        assert refgold.digest(got) == table[key], f"{key}: differs from the reference"
    yield check
    if refgold.RECORD and recorded:
        with open(DIGESTS, "w") as f:
            json.dump({**table, **recorded}, f, indent=0, sort_keys=True)
            f.write("\n")


def test_c2_command_lines(c2, dump_gold):
    for args, exact in ((["-S", "2", "-p", "paf", c2], False), (["-S", "5", "-p", "sg", c2], False), (["-p", "bed", c2], True)):
        rc, out, err = run(OURS, args)
        assert rc == 0, err.decode()[-2000:]
        dump_gold("exact" if exact else "sorted", args, outcome(rc, out, exact), lambda: outcome(*run(REF, args)[:2], exact))
