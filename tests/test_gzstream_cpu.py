"""CPU tier of the streaming GPU gzip decoder (GzStream in miniasm_b200/csrc/gunzip_dev.cu): its segment steps -- which units
chain, where the next segment starts, the history and CRC carried on, all in gzstream.cuh -- run on the host by
tests/hostsim/gzstream_host.cpp over the same inflate.cuh, swept over compressed segment sizes, output caps and chunk sizes on
the corpus of tests/gz_corpus.py, on streams built to put a segment boundary in each awkward place, and under ASan/UBSan."""
import ctypes as C
import gzip
import os
import random
import struct
import subprocess
import sys
import zlib

import pytest

from miniasm_b200 import synth
from tests import gz_corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "gzstream_host.cpp")
BIG = 1 << 62


def _bind(dll):
    dll.gzs_open.restype = C.c_void_p
    dll.gzs_open.argtypes = [C.c_char_p, C.c_uint64, C.c_uint64, C.c_uint64]
    dll.gzs_close.argtypes = [C.c_void_p]
    dll.gzs_rewind.argtypes = [C.c_void_p]
    dll.gzs_fill.restype = C.c_int64
    dll.gzs_fill.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    dll.gzs_counts.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    return dll


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("gzs") / "libgzstream_host.so")
    subprocess.run(["g++", "-std=c++14", "-O2", "-Wall", "-shared", "-fPIC", "-o", out, SRC], check=True)
    return _bind(C.CDLL(out))


@pytest.fixture(scope="module")
def paf(built, paf_dir):
    path = synth.generate("chaos_small", f"{paf_dir}/gz_chaos_small.paf")
    with open(path, "rb") as f:
        data = f.read(150000)
    return data[:data.rindex(b"\n") + 1]


def stream(sim, gz, seg, cap, chunk=0, counts=None, rewind_after=None):
    """All fills of a stream with output room cap (doubled whenever the decoder asks for more, as the ingest's windows grow);
    the concatenated bytes, or None when it rejects.  rewind_after: rewind once after that many fills and start over."""
    h = sim.gzs_open(gz, len(gz), seg, chunk)
    try:
        buf = C.create_string_buffer(max(cap, 1) if cap < BIG else len(gz) * 1100 + 1024)
        room = len(buf) if cap >= BIG else cap
        out, need, fills = [], C.c_uint64(), 0
        while True:
            r = sim.gzs_fill(h, buf, room, C.byref(need))
            if r == -3:
                assert need.value > room
                room = need.value
                buf = C.create_string_buffer(room)
                continue
            if r < 0:
                return None
            if r == 0:
                break
            out.append(buf.raw[:r])
            fills += 1
            if fills == rewind_after:
                sim.gzs_rewind(h)
                out, rewind_after = [], None
        if counts is not None:
            v = (C.c_uint64 * 4)()
            sim.gzs_counts(h, v)
            counts.extend(v)
        return b"".join(out)
    finally:
        sim.gzs_close(h)


SEGS = [1024, 6000, 40000, BIG]
CAPS = [65536, 200000, BIG]


@pytest.mark.parametrize("chunk", [1024, 4096, 65536])
def test_corpus_equals_zlib(sim, paf, chunk):
    for name, gz, want in gz_corpus.valid_corpus(paf):
        for seg in SEGS:
            for cap in CAPS:
                got = stream(sim, gz, min(seg, BIG), cap, chunk)
                assert got == want, (name, seg, cap, chunk)


@pytest.mark.parametrize("cap", [65536, 150000, 1 << 20])
def test_segment_lengths_as_the_device_picks_them(sim, paf, cap):
    """seg = 0: each segment's length from the cap of the fill that chained the one before and the ratio so far, and the room
    memo's early answers, as GzStream does; the bytes still equal zlib's."""
    for name, gz, want in gz_corpus.valid_corpus(paf):
        for chunk in (1024, 0):
            assert stream(sim, gz, 0, cap, chunk) == want, (name, cap, chunk)


def test_bgzf_small_blocks(sim, paf):
    gz = gz_corpus.bgzf(paf, block=3000)
    for seg in (1024, 3000, 9000, BIG):
        for cap in (65536, BIG):
            assert stream(sim, gz, seg, cap, 2048) == paf, (seg, cap)


def test_default_chunks_and_rewind(sim, paf):
    gz = gz_corpus.member(paf * 2, level=1)
    counts = []
    assert stream(sim, gz, 12000, 100000, 0, counts) == paf * 2
    n_seg, n_grow, n_units, n_chain = counts
    assert n_seg > 5 and n_chain >= n_seg - n_grow
    assert stream(sim, gz, 12000, 100000, 0, rewind_after=3) == paf * 2


def _boundaries(gz, seg_list, want, sim):
    for seg in seg_list:
        for cap in (65536, BIG):
            assert stream(sim, gz, seg, cap, 1024) == want, (seg, cap)


def test_boundary_in_header_fields(sim, paf):
    """Segments that end inside a member header with FEXTRA, FNAME, FCOMMENT and FHCRC: the second member's header bytes."""
    a, b = paf[:50000], paf[50000:120000]
    m1 = gz_corpus.member(a, level=1)
    m2 = gz_corpus.member(b, extra=b"BC\x02\x00\x00\x00" + b"x" * 300, name=b"n" * 200 + b".paf", comment=b"c" * 200, hcrc=True, level=1)
    gz = m1 + m2
    h0 = len(m1)
    # the first segment (unit 0 runs to its end) cut inside each field of the second header
    cuts = [h0 + k for k in (1, 5, 11, 100, 320, 450, 700, 760, 761, 762)]
    _boundaries(gz, cuts, a + b, sim)


def test_boundary_in_trailer_and_between_members(sim, paf):
    a, b, c = paf[:40000], paf[40000:90000], paf[90000:150000]
    m1, m2, m3 = (gz_corpus.member(x, level=6) for x in (a, b, c))
    gz = m1 + m2 + m3
    cuts = [len(m1) - k for k in range(1, 9)] + [len(m1), len(m1) + len(m2) - 3, len(m1) + len(m2)]
    _boundaries(gz, cuts, a + b + c, sim)


def test_boundary_in_stored_block(sim, paf):
    data = paf[:200000]
    gz = gz_corpus.member(data, level=0)
    # stored blocks of 64 KiB - 1: cut inside the first block's body and inside the second block's LEN/NLEN
    cuts = [12, 5000, 65535, 65535 + 10 + 3, 65535 + 10 + 5 + 2]
    _boundaries(gz, cuts, data, sim)


class _Bits:
    """LSB-first bit writer (RFC 1951 3.1.1); Huffman codes are written most significant bit first."""
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, x, k):
        self.v |= x << self.n
        self.n += k

    def code(self, c, k):
        self.put(int(format(c, f"0{k}b")[::-1], 2), k)

    def align(self):
        self.n = (self.n + 7) // 8 * 8

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def _far_match_stream(n_match):
    """A stored block of 32 768 bytes, then a dynamic block (one a block-start guess can find) of n_match matches of length 258
    at distance 32 768: zlib never writes that distance."""
    rnd = random.Random(3)
    blk = bytes(rnd.choice(b"ACGT\t\n") for _ in range(32768))
    w = _Bits()
    w.put(0, 1), w.put(0, 2), w.align()                     # stored, not final
    w.put(32768, 16), w.put(32768 ^ 0xffff, 16)
    for x in blk:
        w.put(x, 8)
    w.put(1, 1), w.put(2, 2)                                 # dynamic, final
    w.put(29, 5), w.put(29, 5), w.put(14, 4)                 # 286 literal/length, 30 distance, 18 code-length codes
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1]
    for sym in order:
        w.put(1 if sym in (0, 1) else 0, 3)                  # code-length code: 0 -> '0', 1 -> '1'
    lens = [0] * 286 + [0] * 30
    lens[256] = lens[285] = 1                                # end of block '0', length 258 '1'
    lens[286 + 28] = lens[286 + 29] = 1                      # distance codes 28 '0' and 29 '1'
    for x in lens:
        w.code(x, 1)
    for _ in range(n_match):
        w.code(1, 1), w.code(1, 1), w.put(32768 - 24577, 13)
    w.code(0, 1)
    w.align()
    data = blk * (1 + (n_match * 258 + 32767) // 32768)
    data = data[:32768 + n_match * 258]
    return b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\x03" + w.bytes() + struct.pack("<II", zlib.crc32(data), len(data)), data


def test_match_at_32768_across_a_boundary(sim):
    """A match at distance 32 768 whose source lies in the history carried from the previous segment."""
    gz, data = _far_match_stream(2000)
    assert gzip.decompress(gz) == data
    for seg in list(range(33000, len(gz), 211)) + [BIG]:
        for cap in (32768, 40000, BIG):
            assert stream(sim, gz, seg, cap, 1024) == data, (seg, cap)
    counts = []
    assert stream(sim, gz, 32783 + 1500, BIG, 1024, counts) == data
    assert counts[0] - counts[1] == 2 and counts[3] == 2   # the dynamic block decoded in a segment of its own


def test_crc_spans_many_segments(sim, paf):
    gz = gz_corpus.member(paf, level=1, flush_every=4000)
    counts = []
    assert stream(sim, gz, 8192, 65536, 1024, counts) == paf
    assert counts[0] - counts[1] >= 3 # one member, its CRC carried through at least three segments


def test_trailer_garbage_and_bad_crc_rejected_at_the_end(sim, paf):
    good = gz_corpus.member(paf[:100000], level=1)
    for bad in (good + b"\x1f", good + b"\x1f\x8b\x08\x00", good[:-8] + struct.pack("<I", zlib.crc32(paf[:100000]) ^ 1) + good[-4:]):
        for seg in (1024, 20000, BIG):
            assert stream(sim, bad, seg, 65536, 1024) is None, seg


@pytest.mark.parametrize("chunk", [1024, 65536])
def test_damaged_rejected(sim, paf, chunk):
    for name, gz in gz_corpus.damaged_corpus(paf):
        for seg in (1024, 16384, BIG):
            for cap in (65536, BIG):
                assert stream(sim, gz, seg, cap, chunk) is None, (name, seg, cap)


def test_sanitized_random_segments(paf, tmp_path):
    """ASan/UBSan build: random segment sizes, caps and chunks over the valid and damaged corpus, without a finding."""
    so = str(tmp_path / "libgzstream_asan.so")
    subprocess.run(["g++", "-std=c++14", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-shared", "-fPIC",
                    "-o", so, SRC], check=True)
    script = f"""
import ctypes as C, random, sys
sys.path.insert(0, {ROOT!r})
from tests import gz_corpus
from tests.test_gzstream_cpu import _bind, stream, BIG
L = _bind(C.CDLL({so!r}))
paf = open({str(tmp_path / 'p.paf')!r}, 'rb').read()
rnd = random.Random(17)
valid = gz_corpus.valid_corpus(paf)
for i in range(150):
    name, gz, want = valid[i % len(valid)]
    seg, cap = rnd.choice([rnd.randrange(200, 40000), BIG]), rnd.choice([rnd.randrange(1, 200000), BIG])
    got = stream(L, gz, seg, cap, rnd.choice([1024, 2048, 4096, 0]))
    assert got == want, (name, seg, cap)
for name, gz in gz_corpus.damaged_corpus(paf):
    assert stream(L, gz, rnd.randrange(200, 40000), rnd.randrange(1, 200000), rnd.choice([1024, 4096])) is None, name
print("ok")
"""
    (tmp_path / "p.paf").write_bytes(paf[:60000])
    (tmp_path / "run.py").write_text(script)
    env = dict(os.environ)
    env["LD_PRELOAD"] = subprocess.run(["g++", "-print-file-name=libasan.so"], stdout=subprocess.PIPE, text=True).stdout.strip()
    env["ASAN_OPTIONS"] = "detect_leaks=0"
    r = subprocess.run([sys.executable, str(tmp_path / "run.py")], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                       timeout=1200)
    assert r.returncode == 0 and r.stdout.startswith("ok"), r.stderr[-3000:]
