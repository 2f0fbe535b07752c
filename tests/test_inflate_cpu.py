"""CPU tier of the GPU gzip decoder: the chunk / guess / decode / chain / window / resolve / CRC steps of
miniasm_b200/csrc/gunzip_dev.cu run one chunk after another on the host over the same inflate.cuh (tests/hostsim/
inflate_host.cpp), against zlib on the corpus of tests/gz_corpus.py, and sanitizer-built decodes from arbitrary bit offsets."""
import ctypes as C
import gzip
import os
import random
import subprocess
import sys
import zlib

import pytest

from miniasm_b200 import synth
from tests import gz_corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "inflate_host.cpp")


def _compile(out, flags):
    subprocess.run(["g++", "-std=c++14", "-Wall", "-shared", "-fPIC"] + flags + ["-o", out, SRC], check=True)
    dll = C.CDLL(out)
    dll.gzh_inflate.restype = C.c_int
    dll.gzh_inflate.argtypes = [C.c_char_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t, C.POINTER(C.POINTER(C.c_uint8)),
                                C.POINTER(C.c_size_t), C.POINTER(C.c_uint32)]
    dll.gzh_free.argtypes = [C.c_void_p]
    dll.gzh_decode_at.restype = C.c_int
    dll.gzh_decode_at.argtypes = [C.c_char_p, C.c_size_t, C.c_uint64, C.c_int, C.c_size_t, C.POINTER(C.c_uint64)]
    dll.gzh_guess_at.restype = C.c_int
    dll.gzh_guess_at.argtypes = [C.c_char_p, C.c_size_t, C.c_uint64]
    dll.gzh_crc32.restype = C.c_uint32
    dll.gzh_crc32.argtypes = [C.c_char_p, C.c_size_t, C.c_size_t]
    return dll


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    return _compile(str(tmp_path_factory.mktemp("inf") / "libinflate_host.so"), ["-O2"])


@pytest.fixture(scope="module")
def paf(built, paf_dir):
    path = synth.generate("chaos_small", f"{paf_dir}/gz_chaos_small.paf")
    with open(path, "rb") as f:
        data = f.read(400000)
    return data[:data.rindex(b"\n") + 1]


def inflate(sim, gz, chunk, mode=0, seg=1000):
    out, n, info = C.POINTER(C.c_uint8)(), C.c_size_t(), (C.c_uint32 * 8)()
    rc = sim.gzh_inflate(gz, len(gz), chunk, mode, seg, C.byref(out), C.byref(n), info)
    if rc:
        return rc, None, list(info[:5])
    data = C.string_at(out, n.value)
    sim.gzh_free(out)
    return rc, data, list(info[:5])


@pytest.mark.parametrize("chunk", [1024, 4096, 16384, 65536])
def test_corpus_equals_zlib(sim, paf, chunk):
    for name, gz, want in gz_corpus.valid_corpus(paf):
        assert gzip.decompress(gz) == want, name
        rc, got, info = inflate(sim, gz, chunk)
        assert rc == 0 and got == want, (name, chunk, rc, info)


def test_guesses_are_confirmed(sim, paf):
    """On PAF from gzip -1 nearly every chunk's guess is a true block start (the chain follows it)."""
    gz = gz_corpus.member(paf * 3, level=1)
    rc, got, (n_units, n_chain, n_conf, n_members, n_chunks) = inflate(sim, gz, 4096)
    assert rc == 0 and got == paf * 3 and n_members == 1
    assert n_conf == n_units - 1 and n_units > 5


def test_wrong_and_missing_guesses(sim, paf):
    """Every guess forced to a wrong bit, or no guesses at all: still exact (chunk 0's decode runs to the end)."""
    for name, gz, want in gz_corpus.valid_corpus(paf)[::3]:
        for mode in (1, 2):
            rc, got, info = inflate(sim, gz, 2048, mode)
            assert rc == 0 and got == want, (name, mode, info)
            assert info[1] == 1


def test_weird_names_fail_guesses(sim):
    w = gz_corpus.weird_paf()
    gz = gz_corpus.member(w, level=6)
    rc, got, info = inflate(sim, gz, 1024)
    assert rc == 0 and got == w and info[2] == 0


@pytest.mark.parametrize("chunk", [1024, 65536])
def test_damaged_rejected(sim, paf, chunk):
    for name, gz in gz_corpus.damaged_corpus(paf):
        rc, _, info = inflate(sim, gz, chunk)
        assert rc == -2, (name, info)


def test_crc_join(sim):
    rnd = random.Random(5)
    for n in (0, 1, 7, 1000, 4096, 100003):
        data = bytes(rnd.randrange(256) for _ in range(n))
        for seg in (1, 3, 1000, 65536):
            assert sim.gzh_crc32(data, n, seg) == zlib.crc32(data), (n, seg)


def test_sanitized_random_starts(paf, tmp_path):
    """ASan/UBSan build: decodes from 10^4 random bit offsets of real streams and from random byte strings terminate
    without a finding (a finding aborts the process running them)."""
    so = str(tmp_path / "libinflate_asan.so")
    subprocess.run(["g++", "-std=c++14", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-shared", "-fPIC",
                    "-o", so, SRC], check=True)
    script = f"""
import ctypes as C, random, sys, zlib
sys.path.insert(0, {ROOT!r})
from tests import gz_corpus
L = C.CDLL({so!r})
L.gzh_decode_at.argtypes = [C.c_char_p, C.c_size_t, C.c_uint64, C.c_int, C.c_size_t, C.POINTER(C.c_uint64)]
L.gzh_guess_at.argtypes = [C.c_char_p, C.c_size_t, C.c_uint64]
paf = open({str(tmp_path / 'p.paf')!r}, 'rb').read()
rnd = random.Random(11)
streams = [gz_corpus.member(paf, level=l) for l in (1, 6, 9)] + [gz_corpus.member(paf, level=6, strategy=zlib.Z_FIXED), gz_corpus.bgzf(paf, 30000)]
n = C.c_uint64()
stat = {{}}
for i in range(10000):
    s = streams[i % len(streams)]
    b = rnd.randrange(len(s) * 8)
    r = L.gzh_decode_at(s, len(s), b, 0, 4096, C.byref(n))
    L.gzh_guess_at(s, len(s), b)
    stat[r] = stat.get(r, 0) + 1
for i in range(2000):
    s = bytes(rnd.randrange(256) for _ in range(rnd.randrange(1, 3000)))
    if i % 2: s = b'\\x1f\\x8b\\x08\\x00' + s
    L.gzh_decode_at(s, len(s), rnd.randrange(len(s) * 8) if i % 2 == 0 else 0, i % 2, 512, C.byref(n))
    L.gzh_guess_at(s, len(s), rnd.randrange(len(s) * 8))
print("ok", stat)
"""
    (tmp_path / "p.paf").write_bytes(paf[:100000])
    (tmp_path / "run.py").write_text(script)
    env = dict(os.environ)
    asan = subprocess.run(["g++", "-print-file-name=libasan.so"], stdout=subprocess.PIPE, text=True).stdout.strip()
    env["LD_PRELOAD"] = asan
    env["ASAN_OPTIONS"] = "detect_leaks=0"
    r = subprocess.run([sys.executable, str(tmp_path / "run.py")], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                       timeout=900)
    assert r.returncode == 0 and r.stdout.startswith("ok"), r.stderr[-3000:]
