"""All-vs-all PAF from a layout with repeated sequence: direct and inverted repeats, tandem arrays, circular chromosomes,
plasmids that share an insertion element with the chromosome, and heterozygous regions.

pafgen (miniasm_b200/synth/pafgen.c) samples reads from one linear genome without repeats, so the graphs built from its
PAFs only carry noise topologies.  Here a genome is a list of chromosomes, each linear or circular, each a list of blocks
`(content_id, strand, length)`: a unique block has its own content id, the copies of a repeat share one (an inverted copy
has strand -1), and a heterozygous region is a `Het((id_a, strand, len), (id_b, strand, len))` of which each read takes one
side.  Reads are intervals of one haplotype of one chromosome (on a circle they may wrap past the origin), with lengths,
strand and end jitter drawn as pafgen draws them.

A read is a list of content pieces.  Two reads align wherever they share a piece, on a fixed diagonal and relative
strand; pieces on the same diagonal that touch are one alignment, so an alignment extends through neighbouring pieces for
as long as both reads carry the same content.  Each maximal alignment of at least `min_olap` bp is one PAF line (mapq 255,
`ml = bl / 5`).  This gives internal matches inside repeats, dovetails at repeat boundaries (which make the graph branch)
and containments.  `reads_fasta` writes the reads' bases, drawn at random per content id, so that `-f` sees the layout.

Everything is drawn from numpy's PCG64 seeded by the set's seed: the same set gives the same bytes everywhere.
"""
import hashlib
import os
from collections import defaultdict

import numpy as np


class Het:
    def __init__(self, a, b):
        self.sides = (a, b)


class Layout:
    def __init__(self, chroms, seed, n_reads=None, coverage=30.0, len_min=8000, len_max=12000, jitter=30, min_olap=2000,
                 copies=None):
        """chroms: list of (blocks, circular).  copies: per chromosome, how many times more reads it gets per bp (plasmid copy
        number); 1 by default."""
        self.rng = np.random.default_rng(seed)
        self.chroms, self.len_min, self.len_max, self.jitter, self.min_olap = chroms, len_min, len_max, jitter, min_olap
        self.copies = copies or [1] * len(chroms)
        self.hap = [[self._expand(blocks, h) for h in (0, 1)] for blocks, _ in chroms]
        size = np.array([sum(b[2] for b in self.hap[c][0]) * self.copies[c] for c in range(len(chroms))], dtype=float)
        mean = 0.5 * (len_min + len_max)
        n = n_reads or int(coverage * size.sum() / mean)
        self.reads = self._sample(n, size / size.sum())

    @staticmethod
    def _expand(blocks, h):
        out = []
        for b in blocks:
            out.append(b.sides[h] if isinstance(b, Het) else b)
        return out

    def _sample(self, n, w):
        rng, reads = self.rng, []
        names = rng.permutation(n)
        for k in range(n):
            c = int(rng.choice(len(w), p=w))
            h = int(rng.integers(0, 2))
            blocks, circ = self.hap[c][h], self.chroms[c][1]
            glen = sum(b[2] for b in blocks)
            ln = int(rng.integers(self.len_min, self.len_max + 1))
            ln = min(ln, glen if not circ else glen - 1)
            start = int(rng.integers(0, glen if circ else glen - ln + 1))
            rev = int(rng.integers(0, 2))
            reads.append({"name": f"r{names[k]}", "len": ln, "pieces": self._pieces(blocks, circ, glen, start, ln, rev)})
        return reads

    @staticmethod
    def _pieces(blocks, circ, glen, start, ln, rev):
        """(content_id, sigma, c0, c1, r0, r1): content [c0, c1) of `content_id` lies at read [r0, r1), in the read's own
        orientation when sigma is +1 and reverse-complemented when it is -1."""
        segs, g = [], 0
        for rep in range(2 if circ else 1):
            for cid, strand, bl in blocks:
                segs.append((g, g + bl, cid, strand))
                g += bl
        out = []
        for g0, g1, cid, strand in segs:
            a, b = max(g0, start), min(g1, start + ln)
            if a >= b:
                continue
            c0, c1 = (a - g0, b - g0) if strand > 0 else (g1 - b, g1 - a)
            r0, r1 = a - start, b - start
            sigma = strand
            if rev:
                r0, r1, sigma = ln - r1, ln - r0, -strand
            out.append((cid, sigma, c0, c1, r0, r1))
        return out

    def alignments(self):
        """Maximal alignments (i, j, rel, a0, a1, b0, b1) with i < j and read-coordinate intervals on both reads."""
        by_cid = defaultdict(list)
        for i, r in enumerate(self.reads):
            for p in r["pieces"]:
                by_cid[p[0]].append((i, p))
        seeds = defaultdict(list)
        for cid in sorted(by_cid):
            lst = by_cid[cid]
            for x in range(len(lst)):
                i, (_, sa, ca0, ca1, ra0, ra1) = lst[x]
                for y in range(len(lst)):
                    j, (_, sb, cb0, cb1, rb0, rb1) = lst[y]
                    if j <= i:
                        continue
                    p0, p1 = max(ca0, cb0), min(ca1, cb1)
                    if p0 >= p1:
                        continue
                    a0, a1 = (ra0 + p0 - ca0, ra0 + p1 - ca0) if sa > 0 else (ra1 - (p1 - ca0), ra1 - (p0 - ca0))
                    b0, b1 = (rb0 + p0 - cb0, rb0 + p1 - cb0) if sb > 0 else (rb1 - (p1 - cb0), rb1 - (p0 - cb0))
                    rel = sa * sb
                    key = b0 - a0 if rel > 0 else a0 + b1          # diagonal, or anti-diagonal a + b (half-open ends)
                    seeds[(i, j, rel, key)].append((a0, a1))
        out = []
        for (i, j, rel, key), iv in sorted(seeds.items()):
            iv.sort()
            cur = list(iv[0])
            for a0, a1 in iv[1:] + [(None, None)]:
                if a0 is not None and a0 <= cur[1]:
                    cur[1] = max(cur[1], a1)
                    continue
                s, e = cur
                if rel > 0:
                    out.append((i, j, rel, s, e, s + key, e + key))
                else:
                    out.append((i, j, rel, s, e, key - e, key - s))
                if a0 is not None:
                    cur = [a0, a1]
        return out

    def paf(self):
        rng, lines = self.rng, []
        for i, j, rel, a0, a1, b0, b1 in self.alignments():
            if a1 - a0 < self.min_olap:
                continue
            jt = self.jitter
            if jt:
                a0 += int(rng.integers(0, jt + 1)); a1 -= int(rng.integers(0, jt + 1))
                b0 += int(rng.integers(0, jt + 1)); b1 -= int(rng.integers(0, jt + 1))
            if a0 + 50 >= a1 or b0 + 50 >= b1:
                continue
            q, t = (self.reads[i], self.reads[j])
            qs, qe, ts, te = a0, a1, b0, b1
            if rng.integers(0, 2):
                q, t, qs, qe, ts, te = t, q, b0, b1, a0, a1
            bl = max(qe - qs, te - ts)
            lines.append(f"{q['name']}\t{q['len']}\t{qs}\t{qe}\t{'+' if rel > 0 else '-'}\t{t['name']}\t{t['len']}\t{ts}\t{te}"
                         f"\t{bl // 5}\t{bl}\t255\n")
        return "".join(lines)

    def reads_fasta(self, seed=7):
        rng = np.random.default_rng(seed)
        lens = defaultdict(int)
        for blocks in (b for h in self.hap for b in h):
            for cid, _, bl in blocks:
                lens[cid] = max(lens[cid], bl)
        content = {cid: rng.integers(0, 4, lens[cid]).astype(np.uint8) for cid in sorted(lens)}
        acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
        out = []
        for r in self.reads:
            seq = np.zeros(r["len"], dtype=np.uint8)
            for cid, sigma, c0, c1, r0, r1 in r["pieces"]:
                s = content[cid][c0:c1]
                seq[r0:r1] = s if sigma > 0 else 3 - s[::-1]
            text = acgt[seq].tobytes().decode()
            out.append(f">{r['name']}\n" + "\n".join(text[k:k + 80] for k in range(0, len(text), 80)) + "\n")
        return "".join(out)


# ---- named sets -------------------------------------------------------------------------------------------------------

def _u(cid, ln):
    return (cid, 1, ln)


SETS = {
    # a 5 kb direct repeat in three copies: shorter than every read, so reads span it and the graph branches at its ends
    "direct_short": dict(chroms=[([_u(1, 40000), _u(100, 5000), _u(2, 40000), _u(100, 5000), _u(3, 30000), _u(100, 5000),
                                   _u(4, 25000)], False)], seed=11, len_min=4000, len_max=9000),
    # a 15 kb direct repeat in two copies, longer than the longest read: the repeat collapses into one unitig
    "direct_long": dict(chroms=[([_u(1, 50000), _u(100, 15000), _u(2, 40000), _u(100, 15000), _u(3, 40000)], False)], seed=12),
    # an 8 kb and a 15 kb repeat each with one inverted copy
    "inverted": dict(chroms=[([_u(1, 40000), _u(100, 8000), _u(2, 35000), (100, -1, 8000), _u(3, 30000), _u(101, 15000),
                               _u(4, 30000), (101, -1, 15000), _u(5, 30000)], False)], seed=13),
    # a tandem array of four 3 kb copies (plus an inverted one) between unique flanks
    "tandem": dict(chroms=[([_u(1, 40000)] + [_u(100, 3000)] * 4 + [_u(2, 30000), _u(101, 2500), (101, -1, 2500), _u(101, 2500),
                             _u(3, 30000)], False)], seed=14, len_min=4000, len_max=7000),
    # a circular chromosome and two circular plasmids; the first plasmid carries a 6 kb insertion element that the
    # chromosome also carries (twice, once inverted), longer than most reads, so the element collapses into one unitig
    "plasmids": dict(chroms=[([_u(1, 60000), _u(100, 6000), _u(2, 50000), (100, -1, 6000), _u(3, 40000)], True),
                             ([_u(10, 20000), _u(100, 6000), _u(11, 12000)], True),
                             ([_u(20, 24000)], True)], seed=15, copies=[1, 2, 3], len_min=4000, len_max=8000),
    # a 30 kb heterozygous region covered by 1-2 kb reads: each haplotype is a chain of many reads, so the bubble walk from
    # the region's source visits far more than 64 reads
    "het30k": dict(chroms=[([_u(1, 20000), Het(_u(50, 30000), _u(51, 30000)), _u(2, 20000)], False)], seed=16,
                   len_min=1000, len_max=2000, coverage=30.0, min_olap=500),
}

# options of the reference the 1-2 kb reads need: -s 500 (min_span, and min_ovlp which follows it)
OPTS = {"het30k": {"min_span": 500, "min_ovlp": 500}}
CLI_OPTS = {"het30k": ["-s", "500"]}

# sha256 of each set's PAF: the reference's results for these sets are stored as digests, which stay valid only while the
# generator writes these bytes
SHA256 = {
    "direct_short": "9dbd64cffef426d62f974f50d404652044d37340d43ea1360badec1f05e2e63f",
    "direct_long": "286c217f786dc2f230413231ad089abf5037f1a017dfee2708f7ea99d056337f",
    "inverted": "86259a1ea5a7a01e35a820496c0af94d5a4c4c8488daf3a31ecae66914cdd2f0",
    "tandem": "96ff44c9cf28d2e291ef2e46fd17c4af0e0dcab30a40589df93504edafb3f44e",
    "plasmids": "97f8b1b2ef30afa104c75f09c51b740a1187f7864ebb7fcb76576e87f7645044",
    "het30k": "17d0f969f63de7cdf8f197ef7418e32b00b5556c170796ee68b305694e85cbf7",
}


def opt_for(lib, name):
    o = lib.default_opt()
    for k, v in OPTS.get(name, {}).items():
        setattr(o, k, v)
    return o


def layout(name):
    return Layout(**SETS[name])


def het_reads(name):
    """Names of the reads that lie wholly inside a heterozygous region (on either haplotype)."""
    het = {s[0] for blocks, _ in SETS[name]["chroms"] for b in blocks if isinstance(b, Het) for s in b.sides}
    return {r["name"] for r in layout(name).reads if all(p[0] in het for p in r["pieces"])}


def generate(name, path):
    """Writes the set's PAF to path (if it is not there already with the same bytes) and returns path."""
    text = layout(name).paf().encode()
    if not (os.path.exists(path) and open(path, "rb").read() == text):
        with open(path, "wb") as f:
            f.write(text)
    return path


def sha256(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()
