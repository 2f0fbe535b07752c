"""The windowed ingest (mab_ingest_windowed / mab_ingest_file_windowed, ingest_paf_windowed in ingest_dev.cu): the PAF is taken
from a source in windows and read twice, and must leave what mab_ingest leaves from the resident text -- the hits and names of
the oracle port's ma_hit_read, the same counters, and the very same hit array as mab_ingest (same stable order).  Window edges
(a line ending at, straddling and longer than a window, CRLF split across two windows, a long name whose witness lies in an
earlier window, more names than the first dictionary and name store hold), sources that misbehave, and the whole command line
with MINIASM_B200_INGEST=windowed."""
import ctypes as C
import gzip
import hashlib
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from miniasm_b200 import capi, synth
from miniasm_b200.capi import HIT_DT
from tests import wild_paf
from tests.test_cli_gpu import CLI, REF, _counters, _reads_file, run
from tests.test_ingest_onepass_gpu import boundary_text, canon, oracle, ordinary, overflow_text, parsed_lines, rec, small_texts

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KB, MB = 1 << 10, 1 << 20
WINDOWS = [64 * KB, MB, 64 * MB]     # the smallest, one between, one larger than every text that uses the list


class Source:
    """mab_text_source_t over bytes.  second = what it delivers from the second rewind on (a source that lies);
    rewindable = False: rewind reports -1; short = largest read it answers (a source may deliver less than asked)."""

    def __init__(self, data, second=None, rewindable=True, short=None):
        self.data, self.second, self.rewindable, self.short = data, second, rewindable, short
        self.pos, self.rewinds = 0, 0
        self._keep = (capi.MAB_READ_FN(self._read), capi.MAB_REWIND_FN(self._rewind))
        self.struct = capi.MabTextSource(self._keep[0], self._keep[1], None)

    def _read(self, ud, dst, cap):
        n = min(cap, len(self.data) - self.pos, self.short or cap)
        if n > 0:
            C.memmove(dst, np.frombuffer(self.data, np.uint8, n, self.pos).ctypes.data, n)
            self.pos += n
        return max(n, 0)

    def _rewind(self, ud):
        if not self.rewindable:
            return -1
        self.rewinds += 1
        if self.rewinds == 2 and self.second is not None:
            self.data = self.second
        self.pos = 0
        return 0


def state(prod, ctx):
    n = C.c_size_t(0)
    hp = prod.mab_export_hits(ctx, C.byref(n))
    hits = capi.np_from_ptr(hp, n.value, HIT_DT).copy()
    capi.c_free(hp)
    hits["bl_del"] &= 0x7fffffff
    d = prod.mab_export_dict(ctx)
    names = [(d.contents.seq[i].name, d.contents.seq[i].len) for i in range(d.contents.n_seq)]
    prod.sd_destroy(d)
    st = prod.mab_stats(ctx).contents
    return hits, names, (st.n_lines, st.n_hits_stored, st.n_seq_in)


def resident(prod, data):
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    assert prod.mab_load_paf_text(ctx, data, len(data)) == 0
    prod.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    out = state(prod, ctx)
    prod.mab_destroy(ctx)
    return out


def windowed(prod, data, window, regrow=None, **kw):
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    src = Source(data, **kw)
    assert prod.mab_ingest_windowed(ctx, C.byref(src.struct), window, opt.min_span, opt.min_match, 1) == 0
    out = state(prod, ctx)
    if regrow is not None:                  # how often pass 1 ran again with a larger dictionary or name store
        regrow[window] = prod.mab_stats(ctx).contents.n_name_regrow
    prod.mab_destroy(ctx)
    return out, src


def check(prod, port, data, path, windows=WINDOWS, regrow=None, **kw):
    with open(path, "wb") as f:
        f.write(data)
    w_hits, w_names = oracle(port, path, False)
    r_hits, r_names, r_counters = resident(prod, data)
    assert r_names == w_names and np.array_equal(canon(r_hits), w_hits)
    for window in windows:
        (hits, names, counters), src = windowed(prod, data, window, regrow, **kw)
        assert names == w_names, f"window {window}: read names / lengths differ"
        assert np.array_equal(canon(hits), w_hits), f"window {window}: hits differ ({len(hits)} vs {len(w_hits)})"
        assert counters == (parsed_lines(data), len(w_hits), len(w_names)) == r_counters, f"window {window}: counters {counters}"
        assert hits.tobytes() == r_hits.tobytes(), f"window {window}: not the hit array of mab_ingest"
    return src


# ---- 1. the state of mab_ingest and of the oracle ----------------------------------------------------------------------------
def targets_first_text():
    """names that appear as targets before they ever appear as queries, with another length column there (sd_put keeps the first)"""
    out = []
    for k in range(6000):
        out.append(rec(b"q%d" % (k // 30), b"late%d" % (k % 700), k))
    for k in range(6000):                      # the late names as queries, each with a length column of its own
        r = rec(b"late%d" % (k % 700), b"q%d" % (k % 200), k + 1)
        c = r.split(b"\t")
        c[1] = b"%d" % (20000 + k)
        out.append(b"\t".join(c))
    return b"".join(out)


def tied_first_text():
    """every name is first seen on a line where it is query and target at once, or on one line with another new name, and those
    lines lie ~70 KB apart, i.e. in different 64 KB windows: ids follow line order, query before target"""
    out, k, n = [], 0, 0
    for r in range(40):
        out.append(rec(b"self%d" % r, b"self%d" % r, k))
        out.append(rec(b"a%d" % r, b"b%d" % r, k + 1))
        out.append(rec(b"b%d" % r, b"a%d" % r, k + 2, nf=10))
        k += 3
        n += sum(map(len, out[-3:]))
        while n < (r + 1) * 70 * KB:
            out.append(ordinary(k))
            n += len(out[-1])
            k += 1
    return b"".join(out)


def test_ordinary_lines(prod, port, tmp_path):
    check(prod, port, b"".join(ordinary(k) for k in range(60000)), str(tmp_path / "ordinary.paf"))


@pytest.mark.parametrize("name", list(small_texts()) + ["empty", "newlines_over_windows"])
def test_small_texts(name, prod, port, tmp_path):
    check(prod, port, dict(small_texts(), empty=b"", newlines_over_windows=b"\n" * 200000)[name], str(tmp_path / f"{name}.paf"))


def test_tile_and_chunk_boundaries(prod, port, tmp_path):
    check(prod, port, boundary_text(), str(tmp_path / "boundaries.paf"), windows=[64 * KB, 100 * MB + 8192])


def test_names_first_seen_as_targets(prod, port, tmp_path):
    check(prod, port, targets_first_text(), str(tmp_path / "targets_first.paf"))


def test_tied_first_appearances_in_different_windows(prod, port, tmp_path):
    check(prod, port, tied_first_text(), str(tmp_path / "tied.paf"))


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_wild_corpus(seed, built, prod, port, paf_dir, tmp_path):
    base = synth.generate("-n 800 -s 31 -j 200 -C 200000", f"{paf_dir}/windowed_wild_base.paf")
    path = f"{paf_dir}/windowed_wild{seed}.paf"
    wild_paf.make(base, path, seed)
    check(prod, port, open(path, "rb").read(), str(tmp_path / "wild.paf"))


def test_source_that_answers_short_reads(prod, port, tmp_path):
    check(prod, port, b"".join(ordinary(k) for k in range(20000)), str(tmp_path / "short.paf"), windows=[64 * KB], short=1000)


# ---- 2. window edges ---------------------------------------------------------------------------------------------------------
W = 64 * KB


def pad_to(parts, target):
    """ordinary lines, then one filler line, so that the text is `target` bytes long"""
    k = len(parts)
    while sum(map(len, parts)) + 400 < target:
        parts.append(ordinary(k))
        k += 1
    n = sum(map(len, parts))
    parts.append(b"#" * (target - n - 1) + b"\n")


@pytest.mark.parametrize("kind", ["ends_at_window_end", "straddles", "crlf_split", "bl_across"])
def test_window_edge(kind, prod, port, tmp_path):
    parts = []
    if kind == "ends_at_window_end":
        r = rec(b"edgeq", b"edget", 11)
        pad_to(parts, W - len(r))
        parts.append(r)                                        # its '\n' is the window's last byte
    elif kind == "straddles":
        pad_to(parts, W - 5)
        parts.append(rec(b"edgeq", b"edget", 11))              # the window ends inside its query name
    elif kind == "crlf_split":
        r = rec(b"edgeq", b"edget", 11, end=b"\r\n")
        pad_to(parts, W - len(r) + 1)
        parts.append(r)                                        # '\r' is the window's last byte, '\n' the next one's first
    else:                                                      # 10-column lines whose bl comes from two windows back
        parts.append(rec(b"blq", b"blt", 5))
        for k in range(4000):                                  # ~3 windows of 10-column lines
            parts.append(rec(b"r%d" % (k % 50), b"s%d" % (k % 70), k, nf=10))
    parts += [ordinary(k) for k in range(3000)]
    check(prod, port, b"".join(parts), str(tmp_path / "edge.paf"), windows=[W])


def test_line_longer_than_the_window(prod, port, tmp_path):
    """the windows grow to hold it (here 64 KB -> 512 KB), before and after lines of ordinary length"""
    data = b"".join(ordinary(k) for k in range(3000)) + rec(b"giant", b"read7", 7, tag=b"cg:Z:" + b"9M" * (150 * KB)) + \
        b"".join(ordinary(k) for k in range(3000, 9000))
    check(prod, port, data, str(tmp_path / "giant.paf"), windows=[W])


def test_long_names_with_the_witness_in_an_earlier_window(prod, port, tmp_path):
    """70 001-byte names that differ in their last byte; each is met again windows after its first occurrence"""
    stem = b"N" * 70000
    lines = [rec(stem + b"%d" % (k % 4), stem + b"%d" % ((k + 1) % 4), k) for k in range(12)]
    data = b"".join(ordinary(k) for k in range(500)).join(lines)
    check(prod, port, data, str(tmp_path / "long_names.paf"), windows=[W, MB])


def test_dictionary_and_name_store_grow(prod, port, tmp_path):
    """1.3 M distinct names: more than the first dictionary (2^20 slots) and the first name store (8 MB) hold, so pass 1 runs again"""
    src = check(prod, port, overflow_text(), str(tmp_path / "many_names.paf"), windows=[4 * MB])
    assert src.rewinds >= 3                                    # pass 1 at least twice, then pass 2


# ---- 3. sources that misbehave -----------------------------------------------------------------------------------------------
LIE = """
import ctypes as C, sys
sys.path.insert(0, {root!r})
from miniasm_b200 import capi
from tests.test_ingest_windowed_gpu import Source
from tests.test_ingest_onepass_gpu import ordinary
prod = capi.load_product(strict=False)
prod.set_verbose(0)
data = b"".join(ordinary(k) for k in range(5000))
second = {second}
opt = prod.default_opt()
ctx = prod.mab_create(0)
src = Source(data, second=second)
rc = prod.mab_ingest_windowed(ctx, C.byref(src.struct), 65536, opt.min_span, opt.min_match, 1)
print("returned", rc)
"""


@pytest.mark.parametrize("second", ["data[:len(data) // 2]",                                  # fewer bytes and lines
                                    "data.replace(b'read7\\t', b'reax7\\t')",                 # a name pass 1 never saw
                                    "data.replace(b'read7\\t', b'read8\\t')"],                # other hit counts per read
                         ids=["shorter", "other_name", "other_counts"])
def test_source_that_delivers_other_bytes_after_rewind(second, built):
    r = subprocess.run([sys.executable, "-c", LIE.format(root=ROOT, second=second)], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert r.returncode == 78, (r.returncode, r.stdout, r.stderr[-2000:])
    assert b"delivered a different text after rewinding" in r.stderr and b"returned" not in r.stdout


def test_source_that_cannot_rewind(prod, port, tmp_path):
    data = b"".join(ordinary(k) for k in range(5000))
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    src = Source(data, rewindable=False)
    assert prod.mab_ingest_windowed(ctx, C.byref(src.struct), W, opt.min_span, opt.min_match, 1) == -1
    good = Source(data)                                        # the context is as usable as before
    assert prod.mab_ingest_windowed(ctx, C.byref(good.struct), W, opt.min_span, opt.min_match, 1) == 0
    got = state(prod, ctx)
    prod.mab_destroy(ctx)
    want = resident(prod, data)
    assert got[1] == want[1] and got[2] == want[2] and got[0].tobytes() == want[0].tobytes()


def test_file_source_and_memory_peak(prod, tmp_path):
    """mab_ingest_file_windowed on a plain and on a gzip file; the allocator's high-water mark stays below the resident ingest's"""
    data = b"".join(ordinary(k) for k in range(400000))       # ~40 MB
    path = str(tmp_path / "file.paf")
    with open(path, "wb") as f:
        f.write(data)
    with gzip.open(path + ".gz", "wb", compresslevel=1) as g:
        g.write(data)
    want = resident(prod, data)
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    assert prod.mab_load_paf_file(ctx, path.encode()) == 0
    prod.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    peak_resident = prod.mab_mem_peak(ctx, 0)
    prod.mab_destroy(ctx)
    for fn in [path, path + ".gz"]:
        ctx = prod.mab_create(0)
        assert prod.mab_ingest_file_windowed(ctx, fn.encode(), MB, opt.min_span, opt.min_match, 1) == 0
        peak = prod.mab_mem_peak(ctx, 1)
        got = state(prod, ctx)
        assert got[1] == want[1] and got[2] == want[2] and got[0].tobytes() == want[0].tobytes()
        assert peak + len(data) <= peak_resident, (peak, peak_resident)
        assert prod.mab_mem_peak(ctx, 0) <= peak               # restarted at the current use
        prod.mab_destroy(ctx)
    ctx = prod.mab_create(0)
    assert prod.mab_ingest_file_windowed(ctx, str(tmp_path / "missing.paf").encode(), MB, opt.min_span, opt.min_match, 1) == -1
    prod.mab_destroy(ctx)


# ---- 4. the whole command line -----------------------------------------------------------------------------------------------
WENV = {"MINIASM_B200_INGEST": "windowed", "MINIASM_B200_WINDOW": "65536"}


def cli(args, env=None, stdin=None):
    r = subprocess.run([CLI] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, stdin=stdin, env=dict(os.environ, **(env or {})))
    return r.returncode, r.stdout, r.stderr


@pytest.fixture(scope="module")
def chaos(built, paf_dir):
    return synth.generate("chaos", f"{paf_dir}/windowed_chaos.paf")


@pytest.mark.parametrize("opts", [[], ["-S2", "-p", "bed"], ["-S4", "-p", "paf"], ["-p", "sg"], ["-1"], ["-2"], ["-b"], ["-1", "-2", "-p", "sg"]],
                         ids=lambda o: "_".join(o) or "default")
def test_cli_windowed_equals_resident(opts, chaos):
    rc_r, out_r, err_r = cli(opts + [chaos], {"MINIASM_B200_INGEST": "resident"})
    rc_w, out_w, err_w = cli(opts + [chaos], WENV)
    assert rc_r == 0 and rc_w == 0, err_w.decode()[-2000:]
    assert out_w == out_r
    assert _counters(err_w) == _counters(err_r) and b"[W::" not in err_w
    if os.path.exists(REF):                                    # where the reference was built: its bytes and its progress lines too
        rc, out, err = run(REF, opts + [chaos])
        exact = opts in ([], ["-S2", "-p", "bed"], ["-1"], ["-2"], ["-b"])   # the other dumps depend on the reference's unstable sort
        assert (out == out_w) if exact else (sorted(out.splitlines()) == sorted(out_w.splitlines()))


def test_cli_windowed_gzip_and_reads(chaos, paf_dir):
    gz = f"{paf_dir}/windowed_chaos.paf.gz"
    with open(chaos, "rb") as f, gzip.open(gz, "wb") as g:
        shutil.copyfileobj(f, g)
    reads = _reads_file(chaos, f"{paf_dir}/windowed_reads.fa", "fa_wrap")
    rc_r, out_r, err_r = cli(["-f", reads, chaos], {"MINIASM_B200_INGEST": "resident"})
    assert rc_r == 0 and out_r.startswith(b"S\t") and b"\t*\tLN" not in out_r
    for paf in [chaos, gz]:
        rc_w, out_w, err_w = cli(["-f", reads, paf], WENV)     # (the reads file streams into HBM behind the windows)
        assert rc_w == 0 and out_w == out_r
        assert _counters(err_w) == _counters(err_r)


def test_cli_windowed_is_refused_where_it_does_not_apply(chaos):
    want = cli([chaos])[1]
    rc, out, err = cli(["-R", chaos], WENV)
    assert rc == 0 and out == cli(["-R", chaos])[1] and b"[W::main] MINIASM_B200_INGEST=windowed does not cover -R" in err
    with open(chaos, "rb") as f:
        rc, out, err = cli(["-"], WENV, stdin=f)
    assert rc == 0 and out == want and b"[W::main] MINIASM_B200_INGEST=windowed does not cover standard input" in err
    if len(subprocess.run(["nvidia-smi", "-L"], stdout=subprocess.PIPE).stdout.splitlines()) >= 2:
        rc, out, err = cli([chaos], dict(WENV, MINIASM_B200_GPUS="2"))
        assert rc == 0 and out == want and b"[W::main] MINIASM_B200_INGEST=windowed does not cover MINIASM_B200_GPUS" in err
    rc, out, err = cli([chaos], {"MINIASM_B200_INGEST": "auto"})  # a text that fits stays on the resident path
    assert rc == 0 and out == want and b"[W::" not in err


# ---- 5. full size ------------------------------------------------------------------------------------------------------------
def test_config_3_full_size(built):
    """config 3 (1 M reads, 50 M overlaps, 3.06 GB of text) through a callback source: the reference's GFA digest, and a device
    peak over the ingest that is lower than the resident ingest's by at least the text and bounded by hits + windows + 1 GB"""
    import bench
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "configs.json")))["c3_1m"]
    lib = capi.load_product()
    lib.set_verbose(0)
    opt = lib.default_opt()
    window = 256 * MB
    buf, n_bytes, n_lines, free = bench.generate(1_000_000, 3)
    try:
        assert n_bytes == gold["paf_bytes"]
        ctx = lib.mab_create(0)
        assert lib.mab_load_paf_text(ctx, buf, n_bytes) == 0
        lib.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
        peak_resident = lib.mab_mem_peak(ctx, 0)
        lib.mab_destroy(ctx)
        src = Source((C.c_char * n_bytes).from_address(buf.value))
        ctx = lib.mab_create(0)
        assert lib.mab_ingest_windowed(ctx, C.byref(src.struct), window, opt.min_span, opt.min_match, 1) == 0
        del src
    finally:
        free()
    peak = lib.mab_mem_peak(ctx, 1)
    n_hits = lib.mab_stats(ctx).contents.n_hits_stored
    print(f"config 3 ingest peak: resident {peak_resident / 2**30:.2f} GiB, windowed {peak / 2**30:.2f} GiB ({n_hits} hits)")
    assert peak + n_bytes <= peak_resident
    assert peak <= 64 * n_hits + 2 * window + (1 << 30)
    lib.mab_select(ctx, C.byref(opt), 0, 0, 100)
    lib.mab_layout(ctx, C.byref(opt), 100)
    lib.mab_unitigs(ctx)
    d, sub, ug = lib.mab_export_dict(ctx), lib.mab_export_sub(ctx), lib.mab_export_ug(ctx)
    gfa = lib.print_to_string("ma_ug_print", ug, d, sub)
    lib.ma_ug_destroy(ug), capi.c_free(sub), lib.sd_destroy(d), lib.mab_destroy(ctx)
    assert len(gfa) == gold["gfa_bytes"] and hashlib.sha256(gfa).hexdigest() == gold["gfa_sha256"]
