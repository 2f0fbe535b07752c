"""CPU tier of the read-name collision fixture (tests/golden/name_collisions.json.gz, written by make_name_collisions.py).

* The generator's numpy restatement of name_hash equals the header's own (ingest_dev.cuh, compiled for the host by nvcc).
* Every property the fixture claims holds: the pairs share their 27-bit fragment and their home slot at 2^20 slots, the
  "length" pairs differ in length, the "prefix" pairs differ only after their first 16 bytes, the cluster is homed in its
  window and the foreign names in the same window under the -f table's mask.
* A linear-probing model of every table size the code picks for the cluster shows where the dictionary must overflow and
  where it must not, whatever order the GPU threads insert in.  Two facts about linear probing make that order-free:
    - the set of occupied slots does not depend on the insertion order, and a name never probes past the first slot that
      is still empty at the end, so (distance from its home to that slot) + 1 bounds its probe count in every order;
    - R names homed in W consecutive slots occupy R distinct slots from the window's start on, so the one in the farthest
      slot sits at least R - W slots from its home: with R - W >= the probe limit some insertion has to give up.
"""
import ctypes as C
import gzip
import importlib.util
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "name_collisions.json.gz")
GEN = os.path.join(ROOT, "tests", "golden", "make_name_collisions.py")
SIM_SRC = os.path.join(ROOT, "tests", "hostsim", "namehash_host.cu")

PROBE_LIMIT = 1 << 14        # tab_insert, win_insert, win_find, k_gtab_insert
RTAB_LIMIT = 1 << 16         # k_rtab_insert
FIRST_SEED = 1442695040888963407          # the sharded global table's first re-seed: 0 * 6364136223846793005 + 1442695040888963407
# A table that must hold the cluster keeps every probe run at most half the limit: room for the order the GPU threads happen
# to insert in is already inside the bound, so the margin covers a cluster a little denser than this fixture's (a regenerated
# fixture, or a table rule that rounds down once more).  A table that must overflow does so by this many probes at least.
HOLD_MARGIN = 2
OVERFLOW_MARGIN = 4096


def _load_gen():
    spec = importlib.util.spec_from_file_location("make_name_collisions", GEN)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


gen = _load_gen()


@pytest.fixture(scope="module")
def fx():
    with gzip.open(FIXTURE, "rb") as f:
        return json.load(f)


@pytest.fixture(scope="module")
def host_hash(tmp_path_factory):
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc")
    assert nvcc, "nvcc is needed to compile ingest_dev.cuh for the host"
    so = str(tmp_path_factory.mktemp("namehash") / "libnamehash_host.so")
    subprocess.run([nvcc, "-std=c++17", "-O2", "-shared", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a",
                    "-o", so, SIM_SRC], check=True)
    dll = C.CDLL(so)
    dll.nh_hash_many.restype = None
    dll.nh_hash_many.argtypes = [C.c_char_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p]

    def run(names, seed=0):
        buf = b"".join(names)
        off = np.zeros(len(names) + 1, np.uint64)
        off[1:] = np.cumsum([len(n) for n in names])
        out = np.zeros(len(names), np.uint64)
        dll.nh_hash_many(buf, off.ctypes.data, len(names), seed, out.ctypes.data)
        return out
    return run


def h64(names, seed=0):
    return gen.name_hash_bytes([n.encode() if isinstance(n, str) else n for n in names], seed)


# ---- the restatement ---------------------------------------------------------------------------------------------------------
def test_numpy_hash_equals_the_header(host_hash):
    rng = np.random.default_rng(3)
    names = [b"", b"\x80", b"\xff" * 300, b"c005566097", b"c007283121"]
    names += [bytes(rng.integers(0, 256, int(n), dtype=np.uint8)) for n in rng.integers(0, 301, 3000)]
    names += [bytes(rng.integers(0x80, 256, int(n), dtype=np.uint8)) for n in rng.integers(1, 40, 300)]
    for seed in (0, FIRST_SEED):
        assert np.array_equal(gen.name_hash_bytes(names, seed), host_hash(names, seed)), f"seed {seed}"
    # the batch path the search uses (prefix state + decimal digits) against the per-name path
    for prefix, width in ((b"c", 9), (gen.STEM, 8), (b"vv", 9)):
        lo = 123456
        want = host_hash([prefix + b"%0*d" % (width, i) for i in range(lo, lo + 2000)])
        assert np.array_equal(gen.decimal_hashes(prefix, width, lo, lo + 2000), want)
    # the pair the dictionary's design note quotes
    a, b = host_hash([b"c005566097", b"c007283121"])
    assert (int(a), int(b)) == (0x665724c1f1c5f30c, 0x665724d70b35f30c)


# ---- the fixture -------------------------------------------------------------------------------------------------------------
def test_pairs(fx, host_hash):
    pairs = fx["pairs"]
    assert len(pairs) >= 12
    a = [p["a"].encode() for p in pairs]
    b = [p["b"].encode() for p in pairs]
    ha, hb = host_hash(a), host_hash(b)
    assert len(set(a + b)) == 2 * len(pairs)
    for p, x, y, hx, hy in zip(pairs, a, b, ha, hb):
        hx, hy = int(hx), int(hy)
        assert x != y and hx != hy, p
        assert hx >> 37 == hy >> 37 and hx & gen.M20 == hy & gen.M20, p
        assert p["equal22"] == (hx & gen.M22 == hy & gen.M22), p
        assert not any(c in x + y for c in b"\t\n\r "), p
    kinds = [p["kind"] for p in pairs]
    assert kinds.count("length") >= 4 and kinds.count("prefix") >= 4 and kinds.count("short") >= 1
    for p, x, y in zip(pairs, a, b):
        if p["kind"] == "length":   # (they differ at byte 0 as well: the TAB check after the bytes never decides these pairs)
            assert len(x) != len(y)
        elif p["kind"] == "prefix":
            n = os.path.commonprefix([x, y])
            assert len(x) == len(y) and len(n) >= 20 and len(x) - len(n) <= 9
            assert len(n) >= 16 and x[:16] == y[:16]           # equal in their first 16 bytes: a compare of 16 bytes says "same"


def test_cluster_and_foreign(fx, host_hash):
    w = fx["window"]
    base, width = w["base"], w["width"]
    cl = [n.encode() for n in fx["cluster"]]
    fo = [n.encode() for n in fx["foreign"]]
    assert len(cl) == len(set(cl)) == 30000 and len(fo) == len(set(fo)) >= 200 and not set(cl) & set(fo)
    hc, hf = host_hash(cl), host_hash(fo)
    home = hc & np.uint64(gen.M20)
    assert np.all((home >= base) & (home < base + width))
    frag = hc >> np.uint64(37)
    _, cnt = np.unique(frag, return_counts=True)
    assert (cnt > 1).sum() == fx["n_fragment_groups"] >= 500           # names that take the witness comparison inside the run
    m = fx["foreign_mask"]
    fh = hf & np.uint64(m)
    assert np.all((fh >= (base & m)) & (fh < (base & m) + width))
    assert np.all(((hf & np.uint64(gen.M20)) < base) | ((hf & np.uint64(gen.M20)) >= base + width))


# ---- the probing model -------------------------------------------------------------------------------------------------------
def occupancy(homes, cap):
    """final occupied slots of linear probing (order-free), by inserting in one order through a next-free-slot forest"""
    nxt = {}

    def find(s):
        path = []
        while s in nxt:
            path.append(s)
            s = nxt[s]
        for p in path:
            nxt[p] = s
        return s
    slots = np.empty(len(homes), np.int64)
    for i, h in enumerate(homes.tolist()):
        s = find(h)
        slots[i] = s
        nxt[s] = (s + 1) % cap
    occ = np.zeros(cap, bool)
    occ[slots] = True
    assert occ.sum() == len(homes)
    return occ, slots


def probe_bound(homes, cap):
    """most probes any name takes in any insertion order: (distance from its home to the first slot left empty) + 1"""
    occ, _ = occupancy(homes, cap)
    free = np.nonzero(~occ)[0]
    j = np.searchsorted(free, homes)
    end = np.where(j < len(free), free[np.minimum(j, len(free) - 1)], free[0] + cap)
    return int((end - homes).max()) + 1


def must_overflow_by(homes, cap, base, width):
    """R - W for the R names homed in the W = width slots from base on (circularly): in every order, one of them ends up at
    least R - W slots past its home, i.e. needs R - W + 1 probes"""
    rel = (homes - base) % cap
    return int((rel < width).sum()) - width


def tab_cap(n_lines):            # tab_cap_for (ingest_dev.cu)
    cap = 1 << 20
    while cap < n_lines // 8:
        cap <<= 1
    return cap


def gcap(n):                      # the sharded global table for n distinct names
    c = 1 << 16
    while c < 2 * n + 2:
        c <<= 1
    return c


def rcap(n_seq):                  # dg_ugseq_fill's -f table
    c = 1024
    while c < 2 * n_seq:
        c <<= 1
    return c


@pytest.fixture(scope="module")
def hashes(fx):
    return h64(fx["cluster"]), h64(fx["cluster"], FIRST_SEED), h64(fx["foreign"])


def test_local_table_overflows_at_first_size_and_holds_after_one_growth(fx, hashes):
    h0 = hashes[0]
    w = fx["window"]
    assert tab_cap(1024) == 1 << 20               # a callback source (no size hint), and any text below 192 MiB
    homes20 = (h0 & np.uint64(gen.M20)).astype(np.int64)
    assert must_overflow_by(homes20, 1 << 20, w["base"], w["width"]) >= PROBE_LIMIT + OVERFLOW_MARGIN
    homes22 = (h0 & np.uint64(gen.M22)).astype(np.int64)
    assert probe_bound(homes22, 1 << 22) * HOLD_MARGIN <= PROBE_LIMIT


def test_global_table_overflows_at_seed_0_and_holds_after_one_reseed(fx, hashes):
    h0, h1 = hashes[0], hashes[1]
    cap = gcap(len(fx["cluster"]))
    assert cap == 1 << 16
    homes = (h0 & np.uint64(cap - 1)).astype(np.int64)
    assert must_overflow_by(homes, cap, fx["window"]["base"] % cap, fx["window"]["width"]) >= PROBE_LIMIT + OVERFLOW_MARGIN
    assert probe_bound((h1 & np.uint64(cap - 1)).astype(np.int64), cap) * HOLD_MARGIN <= PROBE_LIMIT


def test_read_table_holds_the_cluster_on_one_long_chain(fx, hashes):
    h0, hf = hashes[0], hashes[2]
    # the layout keeps between 16 385 and 30 000 of the cluster's reads (the GPU test checks that): one mask for all of them
    assert rcap(16385) == rcap(30000) == fx["foreign_mask"] + 1
    cap = rcap(len(fx["cluster"]))
    homes = (h0 & np.uint64(cap - 1)).astype(np.int64)
    assert probe_bound(homes, cap) * HOLD_MARGIN <= RTAB_LIMIT
    occ, slots = occupancy(homes, cap)
    # most layout reads sit away from their home, behind other full hashes: a lookup has to probe past mismatches to find them
    assert (slots != homes).mean() > 0.5
    # every foreign name starts its lookup inside the run, so it ends only at the run's empty end
    fhomes = (hf & np.uint64(cap - 1)).astype(np.int64)
    assert occ[fhomes].all()
    # the same holds for the smallest layout this mask covers: the run is the cluster's, whichever reads it keeps
    sub = homes[: 16385]
    occ_s, _ = occupancy(sub, cap)
    assert occ_s[fhomes].mean() > 0.9
