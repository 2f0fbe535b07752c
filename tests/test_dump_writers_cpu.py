"""CPU tier: the record emitters behind mab_write_paf / mab_write_bed / mab_write_sg (dump_dev.cu), compiled for the CPU through
mab_test_dump_host, on hand-built hits, interval tables, arcs and dictionaries.  The expected bytes are a Python restatement of
print_hits / print_subs (static in the reference's main.c:13-30, so no library exports them) and the reference library's own
ma_sg_print (asm.c:41-55) where oracle/_ref is built, else the product's host ma_sg_print."""
import ctypes as C
import os

import numpy as np
import pytest

from miniasm_b200 import capi
from oracle import loaders

DUMP_PAF, DUMP_BED, DUMP_SG = 0, 1, 2


def i32(x):
    """printf's "%d" of a 32-bit value"""
    x = int(x) & 0xffffffff
    return x - (1 << 32) if x >> 31 else x


def py_paf(hits, names, sub):
    """print_hits, main.c:21-30: the fields are "%d" of 32-bit values; s is the 31-bit field, s + 1 is computed in int and
    e - s in unsigned arithmetic."""
    s = (sub["s_del"] & 0x7fffffff).astype(np.int64)
    e = sub["e"].astype(np.int64)
    iv = [b"%s:%d-%d\t%d" % (n, i32(a + 1), i32(b), i32(b - a)) for n, a, b in zip(names, s.tolist(), e.tolist())]
    q = (hits["qns"] >> np.uint64(32)).astype(np.int64).tolist()
    cols = [(hits["qns"] & np.uint64(0xffffffff)).astype(np.uint32), hits["qe"], hits["ts"], hits["te"],
            hits["ml_rev"] & 0x7fffffff, hits["bl_del"] & 0x7fffffff]
    qs, qe, ts, te, ml, bl = (c.astype(np.uint32).view(np.int32).tolist() for c in cols)
    rev = (hits["ml_rev"] >> 31).tolist()
    t = hits["tn"].astype(np.int64).tolist()
    return b"".join(b"%s\t%d\t%d\t%c\t%s\t%d\t%d\t%d\t%d\t255\n" % (iv[q[i]], qs[i], qe[i], b"+-"[rev[i]], iv[t[i]], ts[i], te[i], ml[i], bl[i])
                    for i in range(len(q)))


def py_bed(names, sub):
    """print_subs, main.c:13-19 (the exported dictionary carries no del flags: sd_squeeze has run)"""
    out = []
    for n, sd, e in zip(names, sub["s_del"].tolist(), sub["e"].tolist()):
        if sd & 0x7fffffff != e:
            out.append(b"%s\t%d\t%d\n" % (n, i32(sd & 0x7fffffff), i32(e)))
    return b"".join(out)


def probe(lib):
    f = lib.dll.mab_test_dump_host
    f.restype = C.c_size_t
    f.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.POINTER(capi.Sdict), C.c_void_p, C.c_void_p, C.c_size_t]

    def run(kind, recs, n, d, sub):
        p = C.c_void_p(recs.ctypes.data) if recs is not None and len(recs) else None
        sp = C.c_void_p(sub.ctypes.data) if sub is not None else None
        size = f(kind, p, n, d, sp, None, 0)
        buf = C.create_string_buffer(max(size, 1))
        assert f(kind, p, n, d, sp, buf, size) == size
        return buf.raw[:size]
    return run


NAMES = [b"", b"x", b"N" * 70000, b"read/17", b"m54_0001/4711/ccs", b"z" * 300]


def hand_built(lib, seed, n_hits, n_arcs):
    rng = np.random.default_rng(seed)
    n = len(NAMES)
    d = lib.sd_init()
    for i, nm in enumerate(NAMES):
        assert lib.sd_put(d, nm, 1000 + i) == i
    sub = np.zeros(n, dtype=capi.SUB_DT)
    sub["s_del"] = [0, 5, 0x7fffffff, 0x80000000 | 7, 0x80000000 | 0x7ffffffe, 123]   # s + 1 wraps to INT_MIN; del bits set
    sub["e"] = [0, 5, 0xfffffff0, 9000, 0x80000001, 0x80000000]                         # rows with s == e; e of 2^31 and more
    hits = np.zeros(n_hits, dtype=capi.HIT_DT)
    big = lambda k: rng.choice([0, 1, 0x7fffffff, 0x80000000, 0xffffffff], k).astype(np.uint64) \
        | (rng.integers(0, 2, k).astype(np.uint64) * rng.integers(0, 1 << 32, k, dtype=np.uint64))
    hits["qns"] = (rng.integers(0, n, n_hits).astype(np.uint64) << np.uint64(32)) | (big(n_hits) & np.uint64(0xffffffff))
    for f in ("qe", "ts", "te", "ml_rev", "bl_del"):
        hits[f] = big(n_hits) & np.uint64(0xffffffff)
    hits["tn"] = rng.integers(0, n, n_hits)
    arcs = np.zeros(n_arcs, dtype=capi.ARC_DT)
    arcs["ul"] = (rng.integers(0, 2 * n, n_arcs).astype(np.uint64) << np.uint64(32)) | (big(n_arcs) & np.uint64(0xffffffff))
    arcs["v"] = rng.integers(0, 2 * n, n_arcs)
    arcs["ol_del"] = big(n_arcs) & np.uint64(0xffffffff)
    return d, sub, hits, arcs


@pytest.mark.parametrize("seed,n_hits,n_arcs", [(1, 0, 0), (2, 1, 1), (3, 500, 400)])
def test_paf_and_bed_emitters_match_print_hits_and_print_subs(built, seed, n_hits, n_arcs):
    prod = capi.load_product(strict=False)
    run = probe(prod)
    d, sub, hits, _ = hand_built(prod, seed, n_hits, n_arcs)
    got = run(DUMP_PAF, hits, len(hits), d, sub)
    assert got == py_paf(hits, NAMES, sub)
    if n_hits > 100:
        assert b"\t-" in got and b":-2147483648-" in got and b"N" * 70000 + b":" in got and b"\tx:6-5\t0\t" in got
    bed = run(DUMP_BED, None, len(NAMES), d, sub)
    assert bed == py_bed(NAMES, sub)
    assert bed.count(b"\n") == 4 and not bed.startswith(b"\t0\t0") and b"x\t" not in bed             # s == e rows print nothing
    assert b"N" * 70000 + b"\t2147483647\t-16\n" in bed
    empty = prod.sd_init()
    assert run(DUMP_BED, None, 0, empty, np.zeros(0, dtype=capi.SUB_DT)) == b""
    prod.sd_destroy(empty), prod.sd_destroy(d)


@pytest.mark.parametrize("with_sub", [True, False])
@pytest.mark.parametrize("seed,n_arcs", [(4, 0), (5, 1), (6, 600)])
def test_sg_emitter_matches_ma_sg_print(built, seed, n_arcs, with_sub):
    prod = capi.load_product(strict=False)
    run = probe(prod)
    d, sub, _, arcs = hand_built(prod, seed, 0, n_arcs)
    sp = C.c_void_p(sub.ctypes.data) if with_sub else None
    g = prod.make_graph(arcs, np.full(len(NAMES), 1000, dtype=np.uint32))
    got = run(DUMP_SG, arcs, len(arcs), d, sub if with_sub else None)
    assert got == prod.print_to_string("ma_sg_print", g, d, sp)
    if os.path.exists(loaders.REFERENCE_SO):
        ref = loaders.load_reference()
        d2 = ref.sd_init()
        for i, nm in enumerate(NAMES):
            ref.sd_put(d2, nm, 1000 + i)
        assert got == ref.print_to_string("ma_sg_print", g, d2, sp)
        ref.sd_destroy(d2)
    if n_arcs > 100:
        assert got.count(b"\n") == n_arcs and b":\tL1:i:-" in got and (b":-2147483648-" in got) == with_sub
    prod.asg_destroy(g), prod.sd_destroy(d)
