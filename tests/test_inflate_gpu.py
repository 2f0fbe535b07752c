"""GPU tier of the gzip decoder (gunzip_dev.cu): the corpus of tests/gz_corpus.py through mab_load_paf_gz and through
mab_load_paf_file (against zlib's own gzopen/gzread loop, damaged files included), the command line on gzipped PAF and
reads files, and config 3 at full size from a gzip -1 stream in memory."""
import ctypes as C
import ctypes.util
import gzip
import hashlib
import json
import os
import subprocess

import pytest

import bench
from miniasm_b200 import capi, synth
from tests import gz_corpus

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "miniasm_b200", "miniasm-b200")
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "configs.json")))


@pytest.fixture(scope="module")
def paf(built, paf_dir):
    path = synth.generate("chaos_small", f"{paf_dir}/gz_chaos_small.paf")
    with open(path, "rb") as f:
        data = f.read(400000)
    return data[:data.rindex(b"\n") + 1]


@pytest.fixture(scope="module")
def lib(prod):
    prod.set_verbose(0)
    return prod


def text_of(lib, ctx):
    n = lib.mab_paf_text(ctx, None, 0)
    buf = C.create_string_buffer(n + 1)
    assert lib.mab_paf_text(ctx, buf, n) == n
    return buf.raw[:n]


def gzread_all(path):
    """What zlib's gzopen/gzread loop returns for a file, damaged or not (the loaders' host route)."""
    z = C.CDLL(ctypes.util.find_library("z"))
    z.gzopen.restype, z.gzopen.argtypes = C.c_void_p, [C.c_char_p, C.c_char_p]
    z.gzread.restype, z.gzread.argtypes = C.c_int, [C.c_void_p, C.c_void_p, C.c_uint]
    z.gzclose.argtypes = [C.c_void_p]
    fp = z.gzopen(path.encode(), b"r")
    out, buf = [], C.create_string_buffer(1 << 20)
    while True:
        r = z.gzread(fp, buf, 1 << 20)
        if r <= 0:
            break
        out.append(buf.raw[:r])
    z.gzclose(fp)
    return b"".join(out)


def test_corpus_through_load_paf_gz(lib, paf):
    ctx = lib.mab_create(0)
    try:
        for name, gz, want in gz_corpus.valid_corpus(paf):
            assert lib.mab_load_paf_gz(ctx, gz, len(gz)) == 0, name
            assert text_of(lib, ctx) == want, name
        for name, gz in gz_corpus.damaged_corpus(paf):
            assert lib.mab_load_paf_gz(ctx, gz, len(gz)) == -2, name
            assert lib.mab_paf_text(ctx, None, 0) == 0, name
        plain = b"not gzip\n"
        assert lib.mab_load_paf_gz(ctx, plain, len(plain)) == -2
    finally:
        lib.mab_destroy(ctx)


def test_corpus_through_load_paf_file(lib, paf, tmp_path):
    ctx = lib.mab_create(0)
    try:
        cases = [(n, g) for n, g, _ in gz_corpus.valid_corpus(paf)] + gz_corpus.damaged_corpus(paf)
        for name, gz in cases:
            path = str(tmp_path / f"{name}.paf.gz")
            with open(path, "wb") as f:
                f.write(gz)
            assert lib.mab_load_paf_file(ctx, path.encode()) == 0, name
            assert text_of(lib, ctx) == gzread_all(path), name
    finally:
        lib.mab_destroy(ctx)


def _cli(args):
    r = subprocess.run([CLI] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout


@pytest.mark.parametrize("name", ["chaos_small", "chaos"])
def test_cli_on_gzipped_paf(name, built, paf_dir):
    path = synth.generate(name, f"{paf_dir}/gzc_{name}.paf")
    data = open(path, "rb").read()
    want = _cli([path])
    variants = {f"l{lvl}": gz_corpus.member(data, level=lvl) for lvl in (1, 6, 9)}
    cut = [0, len(data) // 3, len(data) // 2, len(data)]
    variants["members"] = b"".join(gz_corpus.member(data[a:b], level=1) for a, b in zip(cut, cut[1:]))
    variants["bgzf"] = gz_corpus.bgzf(data)
    for tag, gz in variants.items():
        p = f"{paf_dir}/gzc_{name}_{tag}.paf.gz"
        with open(p, "wb") as f:
            f.write(gz)
        assert _cli([p]) == want, tag


@pytest.mark.parametrize("style,ext", [("fa_wrap", "fa"), ("fq", "fq")])
def test_cli_reads_gz(style, ext, built, paf_dir):
    from tests.test_cli_gpu import _reads_file
    paf = synth.generate("chaos_small", f"{paf_dir}/gzr_chaos_small.paf")
    reads = _reads_file(paf, f"{paf_dir}/gzr_reads.{ext}", style)
    want = _cli(["-f", reads, paf])
    data = open(reads, "rb").read()
    for tag, gz in (("one", gz_corpus.member(data, level=6)), ("multi", b"".join(gz_corpus.member(data[i:i + 300000], level=1)
                                                                                 for i in range(0, len(data), 300000)))):
        p = f"{paf_dir}/gzr_reads_{tag}.{ext}.gz"
        with open(p, "wb") as f:
            f.write(gz)
        assert _cli(["-f", p, paf]) == want, tag


def test_config3_from_gzip_in_memory(lib):
    gold = GOLD["c3_1m"]
    buf, n_bytes, n_lines, free = bench.generate(1_000_000, 3)
    try:
        gz = gzip.compress((C.c_char * n_bytes).from_address(buf.value), compresslevel=1)
    finally:
        free()
    ctx = lib.mab_create(0)
    opt = lib.default_opt()
    assert lib.mab_load_paf_gz(ctx, gz, len(gz)) == 0
    del gz
    assert lib.mab_paf_text(ctx, None, 0) == gold["paf_bytes"]
    lib.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    lib.mab_select(ctx, C.byref(opt), 0, 0, 100)
    lib.mab_layout(ctx, C.byref(opt), 100)
    lib.mab_unitigs(ctx)
    d, sub, ug = lib.mab_export_dict(ctx), lib.mab_export_sub(ctx), lib.mab_export_ug(ctx)
    gfa = lib.print_to_string("ma_ug_print", ug, d, sub)
    lib.ma_ug_destroy(ug), capi.c_free(sub), lib.sd_destroy(d), lib.mab_destroy(ctx)
    assert hashlib.sha256(gfa).hexdigest() == gold["gfa_sha256"]
