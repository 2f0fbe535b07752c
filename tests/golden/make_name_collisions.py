#!/usr/bin/env python
"""Writes tests/golden/name_collisions.json.gz: read names built to collide in the read-name dictionaries of the ingest
(ingest_dev.cu tab_insert / win_insert / win_find, the sharded global table) and of the -f name table (ugseq_dev.cu RTab).

Those tables hash a name with name_hash (ingest_dev.cuh: FNV-1a-64, then the fmix64 finaliser, 0 mapped to 1) and keep,
per slot, a 27-bit fragment h >> 37 and the offset of a witness occurrence; the home slot is h & (cap - 1), and the first
local table has cap = 2^20.  Two different names take the witness comparison only when their fragments are equal and one
probes past the other's slot.  This script hashes a few hundred million candidate names on the CPU and keeps:

  pairs    distinct names equal in h >> 37 and in h & (2^20 - 1) (same fragment, same first home slot), of three kinds:
           "length" (the two names differ in length), "prefix" (a 21-byte PacBio-style stem, equal up to the last 8 bytes)
           and "short"; equal22 marks the pairs whose homes are also equal at 2^22 slots.  The two names of a "length" pair
           differ already in their first byte, so the byte loop of the compare decides them: a compare that dropped its length /
           TAB check would still pass every test.  Only a pair where one name is a prefix of the other reaches that check, and
           finding one is a preimage search of 2^39 or more
  cluster  CLUSTER_N names whose h & (2^20 - 1) lies in [base, base + width), with every fragment-equal group the window
           holds first; base is the last `width` slots of the table, so every probe run wraps past the table's end
  foreign  names outside the cluster homed in the same window under the -f table's mask (foreign_mask)

Deterministic; about a minute and a few GB of RAM.  usage: python tests/golden/make_name_collisions.py
"""
import gzip
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "name_collisions.json.gz")

M20, M22 = (1 << 20) - 1, (1 << 22) - 1
BASE, WIDTH = (1 << 20) - 8192, 8192          # the home window of the cluster at 2^20 slots
CLUSTER_N = 30000
FOREIGN_MASK = (1 << 16) - 1                  # -f table of dg_ugseq_fill for 16 385 .. 32 768 layout reads
FOREIGN_N = 300
STEM = b"m54238_180628_014238/"
BATCH = 1 << 24

FNV_OFF, FNV_PRIME = np.uint64(1469598103934665603), np.uint64(1099511628211)


def fmix64(k):
    k = k.copy()
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xff51afd7ed558ccd)
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xc4ceb9fe1a85ec53)
        k ^= k >> np.uint64(33)
    return k


def fnv_state(prefix, seed=0):
    h = np.uint64(FNV_OFF ^ np.uint64(seed))
    with np.errstate(over="ignore"):
        for c in prefix:
            h = (h ^ np.uint64(c)) * FNV_PRIME
    return h


def finish(h):
    k = fmix64(h)
    k[k == 0] = 1
    return k


def name_hash_bytes(names, seed=0):
    """name_hash of a list of byte strings (any lengths), vectorised per length"""
    out = np.zeros(len(names), np.uint64)
    by_len = {}
    for i, nm in enumerate(names):
        by_len.setdefault(len(nm), []).append(i)
    for ln, idx in by_len.items():
        a = np.frombuffer(b"".join(names[i] for i in idx), np.uint8).reshape(len(idx), ln) if ln else np.zeros((len(idx), 0), np.uint8)
        h = np.full(len(idx), FNV_OFF ^ np.uint64(seed), np.uint64)
        with np.errstate(over="ignore"):
            for j in range(ln):
                h = (h ^ a[:, j].astype(np.uint64)) * FNV_PRIME
        out[np.array(idx)] = finish(h)
    return out


def decimal_hashes(prefix, width, lo, hi):
    """name_hash of prefix + '%0{width}d' % i for i in [lo, hi)"""
    out = np.empty(hi - lo, np.uint64)
    h0 = fnv_state(prefix)
    for s in range(lo, hi, BATCH):
        e = min(s + BATCH, hi)
        i = np.arange(s, e, dtype=np.uint64)
        h = np.full(e - s, h0, np.uint64)
        with np.errstate(over="ignore"):
            for k in range(width - 1, -1, -1):
                d = (i // np.uint64(10 ** k)) % np.uint64(10) + np.uint64(48)
                h = (h ^ d) * FNV_PRIME
        out[s - lo:e - lo] = finish(h)
    return out


class Pop:
    """candidate names prefix + width decimal digits, i in [0, n)"""

    def __init__(self, prefix, width, n):
        self.prefix, self.width, self.n = prefix, width, n
        self.h = decimal_hashes(prefix, width, 0, n)

    def name(self, i):
        return self.prefix + b"%0*d" % (self.width, i)


def equal_groups(key):
    """index groups (sorted by first index) of equal values of key"""
    o = np.argsort(key, kind="stable")
    ks = key[o]
    eq = np.nonzero(ks[1:] == ks[:-1])[0]
    groups = {}
    for j in eq:                       # ks[j] == ks[j + 1]: both join the group keyed by the value
        groups.setdefault(int(ks[j]), set()).update((int(o[j]), int(o[j + 1])))
    return sorted((sorted(g) for g in groups.values()), key=lambda g: g[0])


def pair_key(h):
    return (h >> np.uint64(37)) << np.uint64(20) | (h & np.uint64(M20))


def main():
    pairs = []
    # "short": 10-byte names (the search the dictionary's design note quotes)
    short = Pop(b"c", 9, 1 << 26)
    for g in equal_groups(pair_key(short.h)):
        pairs.append(("short", short.name(g[0]), short.name(g[1])))
    # "length": two populations of 9- and 11-byte names; a pair across them differs in length
    a, b = Pop(b"u", 8, 1 << 25), Pop(b"vv", 9, 1 << 25)
    hab = np.concatenate([a.h, b.h])
    for g in equal_groups(pair_key(hab)):
        nm = [a.name(x) if x < a.n else b.name(x - a.n) for x in g[:2]]
        pairs.append(("length" if len(nm[0]) != len(nm[1]) else "short", nm[0], nm[1]))
    del hab, a, b
    # "prefix": 29-byte names that share their first 21 bytes and differ in the last 8
    stem = Pop(STEM, 8, 1 << 26)
    for g in equal_groups(pair_key(stem.h)):
        pairs.append(("prefix", stem.name(g[0]), stem.name(g[1])))
    del stem
    # cluster: the short names homed in the window, fragment-equal groups first, then the others in index order
    home = short.h & np.uint64(M20)
    win = np.nonzero((home >= np.uint64(BASE)) & (home < np.uint64(BASE + WIDTH)))[0]
    frag_groups = equal_groups(short.h[win] >> np.uint64(37))
    pick = [int(win[x]) for g in frag_groups for x in g]
    chosen = set(pick)
    for x in win:
        if len(pick) >= CLUSTER_N:
            break
        if int(x) not in chosen:
            pick.append(int(x)), chosen.add(int(x))
    pick = pick[:CLUSTER_N]
    cluster = [short.name(i) for i in pick]
    # foreign: homed in the window under the -f mask, outside the 2^20 window (so never a cluster candidate)
    fhome = short.h & np.uint64(FOREIGN_MASK)
    fb = BASE & FOREIGN_MASK
    cand = np.nonzero((fhome >= np.uint64(fb)) & (fhome < np.uint64(fb + WIDTH)) &
                      ((home < np.uint64(BASE)) | (home >= np.uint64(BASE + WIDTH))))[0]
    foreign = [short.name(int(i)) for i in cand[:FOREIGN_N]]

    out_pairs = []
    for kind, x, y in pairs:
        hx, hy = name_hash_bytes([x, y])
        out_pairs.append({"kind": kind, "a": x.decode(), "b": y.decode(), "equal22": bool((hx ^ hy) & np.uint64(M22) == 0)})
    doc = {
        "hash": "name_hash: FNV-1a-64 (seed 0), fmix64, 0 -> 1",
        "window": {"bits": 20, "base": BASE, "width": WIDTH},
        "foreign_mask": FOREIGN_MASK,
        "n_fragment_groups": len(frag_groups),
        "pairs": out_pairs,
        "cluster": [n.decode() for n in cluster],
        "foreign": [n.decode() for n in foreign],
    }
    raw = json.dumps(doc, indent=0, sort_keys=True).encode() + b"\n"
    with open(OUT, "wb") as f:
        f.write(gzip.compress(raw, compresslevel=9, mtime=0))
    kinds = {k: sum(p["kind"] == k for p in out_pairs) for k in ("short", "length", "prefix")}
    print(f"{OUT}: {len(out_pairs)} pairs {kinds}, {sum(p['equal22'] for p in out_pairs)} equal at 2^22; cluster {len(cluster)} "
          f"({len(win)} window names, {len(frag_groups)} fragment-equal groups); foreign {len(foreign)}; {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
