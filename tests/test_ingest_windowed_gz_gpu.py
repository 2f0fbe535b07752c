"""The windowed ingest fed by the streaming GPU gzip decoder (GzStream in gunzip_dev.cu, the device source of ingest_paf_windowed):
mab_ingest_gz_windowed on compressed bytes in memory and mab_ingest_file_windowed on a gzip file must leave exactly what the
resident GPU gzip route (mab_load_paf_gz + mab_ingest) leaves, at window sizes from 64 KiB to larger than the text; a stream the
GPU decoder rejects is refused by mab_ingest_gz_windowed and goes through zlib in mab_ingest_file_windowed; the command line
with MINIASM_B200_INGEST=windowed; config 3 at full size with the device memory it takes."""
import ctypes as C
import gzip
import hashlib
import json
import os
import subprocess
import sys

import pytest

from miniasm_b200 import capi, synth
from tests import gz_corpus
from tests.test_cli_gpu import _counters, _reads_file
from tests.test_inflate_gpu import gzread_all
from tests.test_ingest_windowed_gpu import Source, cli, state

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KB, MB = 1 << 10, 1 << 20
WINDOWS = [64 * KB, MB, 64 * MB]


@pytest.fixture(scope="module")
def paf(built, paf_dir):
    path = synth.generate("chaos_small", f"{paf_dir}/gzw_chaos_small.paf")
    with open(path, "rb") as f:
        data = f.read(400000)
    return data[:data.rindex(b"\n") + 1]


@pytest.fixture(scope="module")
def lib(prod):
    prod.set_verbose(0)
    return prod


def resident_gz(lib, gz):
    opt = lib.default_opt()
    ctx = lib.mab_create(0)
    assert lib.mab_load_paf_gz(ctx, gz, len(gz)) == 0
    lib.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    out = state(lib, ctx)
    lib.mab_destroy(ctx)
    return out


def same(a, b):
    return a[1] == b[1] and a[2] == b[2] and a[0].tobytes() == b[0].tobytes()


def test_valid_corpus_equals_resident(lib, paf):
    opt = lib.default_opt()
    ctx = lib.mab_create(0)
    try:
        for name, gz, _ in gz_corpus.valid_corpus(paf):
            want = resident_gz(lib, gz)
            for window in WINDOWS:
                assert lib.mab_ingest_gz_windowed(ctx, gz, len(gz), window, opt.min_span, opt.min_match, 1) == 0, (name, window)
                assert same(state(lib, ctx), want), (name, window)
    finally:
        lib.mab_destroy(ctx)


def test_damaged_corpus(lib, paf, tmp_path):
    """Refused in memory (the context stays usable); from a file, what zlib's gzread delivers, through the host route."""
    opt = lib.default_opt()
    good = gz_corpus.member(paf, level=1)
    want_good = resident_gz(lib, good)
    ctx = lib.mab_create(0)
    try:
        for name, gz in gz_corpus.damaged_corpus(paf):
            for window in (64 * KB, 64 * MB):
                assert lib.mab_ingest_gz_windowed(ctx, gz, len(gz), window, opt.min_span, opt.min_match, 1) == -2, (name, window)
                assert len(state(lib, ctx)[0]) == 0, name
            assert lib.mab_ingest_gz_windowed(ctx, good, len(good), MB, opt.min_span, opt.min_match, 1) == 0
            assert same(state(lib, ctx), want_good), name
        path = str(tmp_path / "good.paf.gz")
        with open(path, "wb") as f:
            f.write(good)
        env = dict(os.environ, MAB_TRACE="1")
        script = (f"import sys; sys.path.insert(0, {ROOT!r}); from miniasm_b200 import capi; L = capi.load_product(); L.set_verbose(0); "
                  f"o = L.default_opt(); c = L.mab_create(0); "
                  f"sys.exit(L.mab_ingest_file_windowed(c, {path.encode()!r}, 65536, o.min_span, o.min_match, 1))")
        r = subprocess.run([sys.executable, "-c", script], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        assert r.returncode == 0 and b"[T::gzstream] mab_ingest_file_windowed: rc 0," in r.stderr, r.stderr[-2000:]  # the GPU route, not zlib
        plain = b"not gzip\n"
        assert lib.mab_ingest_gz_windowed(ctx, plain, len(plain), MB, opt.min_span, opt.min_match, 1) == -2
        for name, gz in gz_corpus.damaged_corpus(paf)[::4] + gz_corpus.damaged_corpus(paf)[-8:]:
            path = str(tmp_path / f"{name}.paf.gz")
            with open(path, "wb") as f:
                f.write(gz)
            src = Source(gzread_all(path))
            assert lib.mab_ingest_windowed(ctx, C.byref(src.struct), 64 * KB, opt.min_span, opt.min_match, 1) == 0
            want = state(lib, ctx)
            assert lib.mab_ingest_file_windowed(ctx, path.encode(), 64 * KB, opt.min_span, opt.min_match, 1) == 0, name
            assert same(state(lib, ctx), want), name
    finally:
        lib.mab_destroy(ctx)


WENV = {"MINIASM_B200_INGEST": "windowed", "MINIASM_B200_WINDOW": "65536"}


@pytest.fixture(scope="module")
def chaos(built, paf_dir):
    return synth.generate("chaos", f"{paf_dir}/gzw_chaos.paf")


@pytest.mark.parametrize("tag", ["l1", "l6", "l9", "members", "bgzf"])
def test_cli_windowed_gzip(tag, chaos, paf_dir):
    data = open(chaos, "rb").read()
    if tag.startswith("l"):
        gz = gz_corpus.member(data, level=int(tag[1:]))
    elif tag == "members":
        cut = [0, len(data) // 3, len(data) // 2, len(data)]
        gz = b"".join(gz_corpus.member(data[a:b], level=1) for a, b in zip(cut, cut[1:]))
    else:
        gz = gz_corpus.bgzf(data)
    path = f"{paf_dir}/gzw_chaos_{tag}.paf.gz"
    with open(path, "wb") as f:
        f.write(gz)
    reads = _reads_file(chaos, f"{paf_dir}/gzw_reads.fa", "fa_wrap")
    for extra in ([], ["-f", reads]):
        rc_r, out_r, err_r = cli(extra + [chaos], {"MINIASM_B200_INGEST": "resident"})
        rc_w, out_w, err_w = cli(extra + [path], WENV)
        assert rc_r == 0 and rc_w == 0, err_w.decode()[-2000:]
        assert out_w == out_r, extra
        assert _counters(err_w) == _counters(err_r) and b"[W::" not in err_w, extra


def test_config_3_gzip_full_size(built):
    """config 3 as gzip -1 in memory at the default window: the reference's GFA digest, and a device peak over the ingest below
    the resident gzip route's by at least the text and within hits + windows + the decoder's scratch + 1 GB"""
    import bench
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "configs.json")))["c3_1m"]
    lib = capi.load_product()
    lib.set_verbose(0)
    opt = lib.default_opt()
    window = 1 << 30                      # the default for gzip (0)
    buf, n_bytes, n_lines, free = bench.generate(1_000_000, 3)
    try:
        assert n_bytes == gold["paf_bytes"]
        gz = gzip.compress((C.c_char * n_bytes).from_address(buf.value), compresslevel=1)
    finally:
        free()
    ctx = lib.mab_create(0)
    assert lib.mab_load_paf_gz(ctx, gz, len(gz)) == 0
    lib.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    peak_resident = lib.mab_mem_peak(ctx, 0)
    lib.mab_destroy(ctx)
    ctx = lib.mab_create(0)
    assert lib.mab_ingest_gz_windowed(ctx, gz, len(gz), 0, opt.min_span, opt.min_match, 1) == 0
    del gz
    peak = lib.mab_mem_peak(ctx, 1)
    n_hits = lib.mab_stats(ctx).contents.n_hits_stored
    seg = window + (16 << 10)                     # the longest segment; its chunks are 64 KiB (gzs_chunk_for)
    scratch = int(seg * (2 + 96 / 64))            # the decoder's scratch, S x (2 + 96 KiB / C) (gunzip_dev.cuh)
    print(f"config 3 gzip ingest peak: resident {peak_resident / 2**30:.2f} GiB, windowed {peak / 2**30:.2f} GiB ({n_hits} hits)")
    assert peak < peak_resident - n_bytes
    assert peak <= 64 * n_hits + 2 * window + scratch + (1 << 30)
    lib.mab_select(ctx, C.byref(opt), 0, 0, 100)
    lib.mab_layout(ctx, C.byref(opt), 100)
    lib.mab_unitigs(ctx)
    d, sub, ug = lib.mab_export_dict(ctx), lib.mab_export_sub(ctx), lib.mab_export_ug(ctx)
    gfa = lib.print_to_string("ma_ug_print", ug, d, sub)
    lib.ma_ug_destroy(ug), capi.c_free(sub), lib.sd_destroy(d), lib.mab_destroy(ctx)
    assert len(gfa) == gold["gfa_bytes"] and hashlib.sha256(gfa).hexdigest() == gold["gfa_sha256"]
