"""Symmetric string graphs built directly from topological motifs, for the cleaning passes and the unitig stage.

`ma_sg_gen` on pafgen's single linear genome only ever yields noise topologies (jitter bubbles, tips, short loops).  The
graphs here are assembled from seeded motifs instead: cycles, figure-eights, nested and chained bubbles, bubbles at the
distance bound, tips at the extension bound, bi-loops with every order of their two overlaps, internal sequences, vertices
with arcs to both strands of a read, walks that return to their source or reach its other strand, deleted reads and reads
without arcs, and a dense graph where every pair of reads overlaps.

Vertices are oriented reads, `2*read + strand`.  Every arc u->v is emitted with its complement v^1->u^1; the overlap `ol` is
shared and each arc's length is its source read's length minus `ol`, as `ma_sg_gen` writes them.  No read has an arc to
itself and no pair (u, v) has two arcs.

`build(name)` returns (arcs, seq, params): `params` holds the `max_ext` and `bub_dist` the passes should run with.

Left out: nothing the reference asserts on.  Every graph here is symmetric and free of multi-arcs, so asg_bub_pop1's
`t->r > 0` and `S.n == 1` (asg.c:341) hold, and asg_cut_biloop only reaches its `w != UINT32_MAX` (asg.c:288) on a vertex
whose complement has exactly one live arc, which always names a w.
"""
import numpy as np

from miniasm_b200.capi import ARC_DT, DEL

MAX_EXT, BUB_DIST = 4, 50000          # the reference's defaults (ma_opt_init)


class Graph:
    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.lens, self.dels, self.arcs = [], set(), {}

    def read(self, ln=None):
        self.lens.append(int(ln if ln is not None else self.rng.integers(8000, 12001)))
        return 2 * (len(self.lens) - 1)

    def reads(self, k, ln=None):
        return [self.read(ln) for _ in range(k)]

    def link(self, u, v, l=None):
        """u->v with length l (u's read length minus the overlap) and its complement; a pair already linked is left alone."""
        assert u >> 1 != v >> 1, "ma_sg_gen never links a read to itself"
        lu, lv = self.lens[u >> 1], self.lens[v >> 1]
        if (u, v) in self.arcs:
            return
        if l is None:
            l = lu - int(self.rng.integers(min(lu, lv) // 2, min(lu, lv) - 300))
        ol = lu - l
        assert 0 < ol < lv, (u, v, l)
        self.arcs[(u, v)] = (l, ol)
        self.arcs[(v ^ 1, u ^ 1)] = (lv - ol, ol)

    def chain(self, vs, l=None):
        for a, b in zip(vs, vs[1:]):
            self.link(a, b, l)

    def delete(self, v):
        self.dels.add(v >> 1)

    def arrays(self):
        rows = [((u << 32) | l, v, ol) for (u, v), (l, ol) in self.arcs.items()]
        arcs = np.array(rows, dtype=ARC_DT) if rows else np.zeros(0, dtype=ARC_DT)
        arcs = arcs[self.rng.permutation(len(arcs))]       # asg_cleanup sorts them
        seq = np.array(self.lens, dtype=np.uint32)
        for r in self.dels:
            seq[r] |= DEL
        return arcs, seq


# ---- motifs: each takes the graph and returns (entry, exit) vertices so that motifs can be strung together -------------

def m_path(g, k=3):
    vs = g.reads(k)
    g.chain(vs)
    return vs[0], vs[-1]


def m_cycle(g, k=None):
    k = k or int(g.rng.integers(2, 6))
    vs = g.reads(k)
    g.chain(vs + [vs[0]])
    return vs[0], vs[-1]


def m_figure_eight(g):
    hub = g.read()
    a, b = g.reads(2), g.reads(3)
    g.chain([hub] + a + [hub])
    g.chain([hub] + b + [hub])
    return hub, b[-1]


def m_bubble(g, na=1, nb=2, la=None, lb=None):
    s, t = g.read(), g.read()
    g.chain([s] + g.reads(na) + [t], la)
    g.chain([s] + g.reads(nb) + [t], lb)
    return s, t


def m_nested_bubble(g):
    s, t = g.read(), g.read()
    g.chain([s, g.read(), t])
    i, o = m_bubble(g)
    g.link(s, i), g.link(o, t)
    return s, t


def m_bubble_chain(g, k=4):
    ends = g.reads(k + 1)
    for a, b in zip(ends, ends[1:]):
        g.chain([a, g.read(), b])
        g.chain([a, g.read(), g.read(), b])
    return ends[0], ends[-1]


def m_bubble_at_dist(g, dist, delta):
    """A bubble whose longer branch reaches its sink at distance dist+delta from the source: the walk's `d + l > max_dist`
    test on either side of the bound."""
    s, t = g.read(20000), g.read(20000)
    a, b = g.read(20000), g.read(20000)
    g.chain([s, a, t], 1000)
    far = dist + delta
    g.link(s, b, far // 2)
    g.link(b, t, far - far // 2)
    return s, t


def m_tip(g, k):
    """A branching vertex with a dead-end chain of k reads hanging off it."""
    x, y = g.read(), g.read()
    g.link(x, y)
    tip = g.reads(k)
    g.chain([x] + tip)
    return x, y


def m_biloop(g, cmp):
    """w->v, w->x and v->c->x' with x' branching again: asg_cut_biloop drops w->x iff ov > ox (asg.c:274-306)."""
    w, v, c, x, z = g.reads(5, 10000)
    l_v = 4000
    l_x = {">": 5000, "<": 3000, "=": 4000}[cmp]                   # ol = 10000 - l
    g.link(w, v, l_v)
    g.link(w, x, l_x)
    g.chain([v, c, x ^ 1])
    g.link(x ^ 1, z)
    return w, z


def m_internal(g, k=2):
    """a->v->...->e->f with a and f branching on either side: a short internal sequence (asg_cut_internal)."""
    a, b, f, h = g.reads(4)
    mid = g.reads(k)
    g.chain([a] + mid + [f])
    g.link(a, b), g.link(h, f)
    return a, f


def m_both_strands(g):
    """u has arcs to both w and w^1."""
    u, w, y = g.reads(3)
    g.link(u, w), g.link(u, w ^ 1)
    g.link(w, y)
    return u, y


def m_back_to_source(g):
    """A bubble source whose one branch comes back to it (w == v0, asg.c:377)."""
    s, a, b, t = g.reads(4)
    g.chain([s, a, s])
    g.chain([s, b, t])
    return s, t


def m_to_other_strand(g):
    """A bubble source whose branch reaches its own other strand (an inverted repeat's hairpin)."""
    s, a, b, t = g.reads(4)
    g.chain([s, a, s ^ 1])
    g.chain([s, b, t])
    return s, t


def m_isolated(g, k=3, deleted=2):
    """Reads without arcs, and deleted reads that still have arcs until asg_cleanup drops them."""
    g.reads(k)
    dv = g.reads(deleted)
    x, y = m_path(g, 2)
    for d in dv:
        g.link(x, d)
        g.delete(d)
    return x, y


def dense(n=31, ln=10000, step=300):
    """n reads of ln bp starting every `step` bp, every pair overlapping and nothing transitively reduced: the walk from read
    0 scans all n(n-1)/2 arcs of the forward strand, far more than 4 per vertex."""
    g = Graph(0)
    vs = g.reads(n, ln)
    for i in range(n):
        for j in range(i + 1, n):
            g.link(vs[i], vs[j], step * (j - i))
    return g


MOTIFS = {
    "cycle": lambda g: m_cycle(g),
    "figure8": m_figure_eight,
    "bubble": lambda g: m_bubble(g),
    "nested": m_nested_bubble,
    "bubble_chain": lambda g: m_bubble_chain(g),
    "tip": lambda g: m_tip(g, int(g.rng.integers(MAX_EXT - 1, MAX_EXT + 2))),
    "biloop": lambda g: m_biloop(g, "<>="[int(g.rng.integers(0, 3))]),
    "internal": lambda g: m_internal(g, int(g.rng.integers(1, 4))),
    "both_strands": m_both_strands,
    "back_to_source": m_back_to_source,
    "to_other_strand": m_to_other_strand,
    "isolated": m_isolated,
}


def _single(motif, **kw):
    def make():
        g = Graph(1)
        a, b = motif(g, **kw) if kw else motif(g)
        x, y = g.read(), g.read()                 # unique flanks, so that the motif sits inside a longer layout
        g.link(x, a), g.link(b, y)
        return g, {}
    return make


def _at_dist(delta):
    def make():
        g = Graph(2)
        s, t = m_bubble_at_dist(g, 30000, delta)
        x, y = g.read(20000), g.read(20000)       # the sink needs an arc of its own, or the walk ends at a tip
        g.link(x, s), g.link(t, y)
        return g, {"bub_dist": 30000}
    return make


def _soup(seed, n_motifs=12, extra=6):
    """Random motifs strung into one component, plus a few random extra arcs between them."""
    def make():
        g = Graph(seed)
        names = sorted(MOTIFS)
        prev = None
        for _ in range(n_motifs):
            a, b = MOTIFS[names[int(g.rng.integers(0, len(names)))]](g)
            if prev is not None and prev >> 1 != a >> 1:
                g.link(prev, a)
            prev = b
        nv = 2 * len(g.lens)
        for _ in range(extra):
            u, v = (int(x) for x in g.rng.integers(0, nv, 2))
            if u >> 1 != v >> 1:
                g.link(u, v)
        return g, {}
    return make


CASES = {
    "cycle2": _single(m_cycle, k=2),
    "cycle5": _single(m_cycle, k=5),
    "figure8": _single(m_figure_eight),
    "nested_bubble": _single(m_nested_bubble),
    "bubble_chain": _single(m_bubble_chain),
    "bubble_dist_under": _at_dist(-1),
    "bubble_dist_exact": _at_dist(0),
    "bubble_dist_over": _at_dist(1),
    "tip_short": _single(m_tip, k=MAX_EXT - 1),
    "tip_bound": _single(m_tip, k=MAX_EXT),
    "tip_long": _single(m_tip, k=MAX_EXT + 1),
    "biloop_ov_gt_ox": _single(m_biloop, cmp=">"),
    "biloop_ov_lt_ox": _single(m_biloop, cmp="<"),
    "biloop_ov_eq_ox": _single(m_biloop, cmp="="),
    "internal1": _single(m_internal, k=1),
    "internal3": _single(m_internal, k=3),
    "both_strands": _single(m_both_strands),
    "back_to_source": _single(m_back_to_source),
    "to_other_strand": _single(m_to_other_strand),
    "isolated_and_deleted": _single(m_isolated),
    "dense31": lambda: (dense(), {}),
    **{f"soup{s}": _soup(s) for s in range(1, 9)},
    "soup_big": _soup(99, n_motifs=120, extra=40),
}


def build(name):
    g, params = CASES[name]()
    arcs, seq = g.arrays()
    return arcs, seq, {"max_ext": params.get("max_ext", MAX_EXT), "bub_dist": params.get("bub_dist", BUB_DIST)}
