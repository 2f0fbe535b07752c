"""The one-pass parse (k_parse_tiles, ingest_dev.cu) on hand-built PAF text: lines that straddle the 8 KB tiles and the 64 MB
chunks of the streamed ingest, lines longer than a tile and than a chunk, CRLF ends, empty lines, no final newline, a text of
only newlines, 10-field lines that take bl from the line before a tile boundary, and more names than the first dictionary holds.
Every entry point (mab_ingest, mab_load_ingest_text, -R, a one-rank sharded ingest resident and streamed) must leave the hits,
names and counters of the oracle port's ma_hit_read."""
import ctypes as C

import numpy as np
import pytest

from miniasm_b200 import capi
from miniasm_b200.capi import HIT_DT

pytestmark = pytest.mark.gpu

TILE = 8192          # PT_TILE
CHUNK = 64 << 20     # chunk of the streamed ingest
ROUTES = ["ingest", "stream", "nocont", "shard", "shard_stream"]


def rec(q, t, k, nf=12, tag=b"", end=b"\n", strand=b"+"):
    """one PAF line that passes the default store filter (spans >= 2000, ml >= 100); nf = 10, 11 or 12 columns (+ tag)"""
    c = [q, b"%d" % (9000 + k % 997), b"%d" % (k % 500), b"%d" % (5000 + k % 3000), strand, t, b"%d" % (9500 + k % 991),
         b"%d" % (k % 700), b"%d" % (6000 + k % 2000), b"%d" % (1000 + k % 900)]
    if nf >= 11:
        c.append(b"%d" % (4000 + k % 1500))
    if nf >= 12:
        c.append(b"255")
    if tag:
        c.append(tag)
    return b"\t".join(c) + end


def ordinary(k, n_reads=3000):
    """the k-th line of a stream of lines naming n_reads reads: query-sorted, a few 10-field, CRLF and empty lines among them"""
    q, t = b"read%d" % (k // 40 % n_reads), b"read%d" % ((k * 7919 + 13) % n_reads)
    if k % 97 == 5:
        return b"\n"
    return rec(q, t, k, nf=10 if k % 23 == 3 else 12, tag=b"tp:A:P" if k % 5 == 0 else b"", end=b"\r\n" if k % 31 == 7 else b"\n",
               strand=b"-" if k % 3 == 0 else b"+")


class Text:
    def __init__(self):
        self.parts, self.n, self.k = [], 0, 0

    def add(self, s):
        self.parts.append(s)
        self.n += len(s)

    def fill_to(self, target, slack=400):
        """ordinary lines up to a little before `target`, then one filler line (fewer than 10 columns) ending at `target`"""
        while self.n + slack < target:
            self.add(ordinary(self.k))
            self.k += 1
        assert target - self.n >= 1
        self.add(b"#" * (target - self.n - 1) + b"\n")

    def at_boundary(self, b, kind):
        """place a line so that byte b (the first byte of a tile or chunk) falls as `kind` says"""
        k = self.k
        self.k += 1
        r = rec(b"bnd%d" % k, b"read%d" % (k % 3000), k)
        if kind == "name":                 # inside the query name
            self.fill_to(b - 3)
            self.add(r)
        elif kind == "number":             # inside the query length
            self.fill_to(b - (r.index(b"\t") + 2))
            self.add(r)
        elif kind == "nl_before":          # the '\n' is the tile's last byte: the next line starts the next tile
            self.fill_to(b - len(r))
            self.add(r)
        elif kind == "nl_at":              # the '\n' is the next tile's first byte
            self.fill_to(b - len(r) + 1)
            self.add(r)
        elif kind == "crlf":               # '\r' ends the tile, '\n' starts the next one
            r = rec(b"crlf%d" % k, b"read%d" % (k % 3000), k, end=b"\r\n")
            self.fill_to(b - len(r) + 1)
            self.add(r)
        elif kind == "bl":                 # a 12-column line ends the tile, 10-column lines start the next one
            r11 = rec(b"blq%d" % k, b"read%d" % (k % 3000), k)
            self.fill_to(b - len(r11))
            self.add(r11)
            self.add(rec(b"blt%d" % k, b"read%d" % ((k + 1) % 3000), k + 1, nf=10))
            self.add(rec(b"blu%d" % k, b"read%d" % ((k + 2) % 3000), k + 2, nf=10))
        elif kind == "long_tile":          # a line longer than a tile (a long tag), and a long name, across the boundary
            self.fill_to(b - 100)
            self.add(rec(b"longtag%d" % k, b"read%d" % (k % 3000), k, tag=b"cg:Z:" + b"7M" * (3 * TILE)))
            self.add(rec(b"N" * (2 * TILE) + b"%d" % k, b"read%d" % (k % 3000), k))
        else:
            raise ValueError(kind)

    def bytes(self):
        return b"".join(self.parts)


KINDS = ["name", "number", "nl_before", "nl_at", "crlf", "bl", "long_tile"]


def boundary_text():
    """~200 MB: every kind at several tile boundaries of the first chunk, then name / number / '\n' at the three chunk boundaries"""
    t = Text()
    bounds = [(TILE * m, KINDS[i % len(KINDS)]) for i, m in enumerate([1, 2, 3, 4, 5, 6, 7, 9, 12, 17, 40, 41, 100, 1000, 1001, 4095, 8190])]
    bounds += [(CHUNK - TILE, "bl"), (CHUNK, "nl_before"), (CHUNK + TILE, "crlf"), (2 * CHUNK, "name"), (3 * CHUNK, "number"),
               (3 * CHUNK + TILE, "nl_at")]
    for b, kind in bounds:
        t.at_boundary(max(b, (t.n + 1000 + TILE - 1) // TILE * TILE), kind)   # (a long line may have passed the boundary: the next free one)
    t.fill_to(t.n + 100000)
    return t.bytes()


def small_texts():
    lines = [ordinary(k) for k in range(3000)]
    body = b"".join(lines)
    return {
        "crlf_everywhere": body.replace(b"\r\n", b"\n").replace(b"\n", b"\r\n") + b"\r\n\r\n\r",
        "empty_lines": b"\n\n" + body.replace(b"\n", b"\n\n\n") + b"\n\n",
        "no_final_newline": body + rec(b"lastq", b"read1", 1, end=b""),
        "only_newlines": b"\n" * 20000,
        "single_line": rec(b"q", b"t", 5, end=b""),
        "one_cr": b"\r",
        "bl_first_line_10": rec(b"q0", b"t0", 1, nf=10) + body,
    }


def chunk_line_text():
    """a line longer than a chunk: the streamed ingest falls back to the resident parse"""
    head = b"".join(ordinary(k) for k in range(20000))
    return head + rec(b"giant", b"read7", 7, tag=b"cg:Z:" + b"9M" * (CHUNK // 2 + 4096)) + b"".join(ordinary(k) for k in range(20000, 40000))


def overflow_text():
    """more distinct names (1.3 M) than the first dictionary of this text's size holds (2^20 slots): the parse runs again"""
    n = 650000
    return b"".join(b"q%d\t9000\t0\t5000\t+\tt%d\t9000\t0\t5000\t3000\t5000\t0\n" % (i, i) for i in range(n))


def parsed_lines(data):
    """lines with at least 10 TAB-separated columns (what ma_hit_read counts as read)"""
    n = 0
    for ln in data.split(b"\n")[: -1 if data.endswith(b"\n") else None]:
        if len(ln) > 1 and ln.endswith(b"\r"):
            ln = ln[:-1]
        n += ln.count(b"\t") >= 9
    return n


def canon(h):
    h = h.copy()
    h["bl_del"] &= 0x7fffffff
    return np.sort(h, order=["qns", "tn", "qe", "ts", "te", "ml_rev", "bl_del"])


def oracle(port, path, nocont):
    opt = port.default_opt()
    excl = port.ma_hit_no_cont(path.encode(), opt.min_span, opt.min_match, opt.max_hang, opt.int_frac) if nocont else None
    d = port.sd_init()
    n = C.c_size_t(0)
    hp = port.ma_hit_read(path.encode(), opt.min_span, opt.min_match, d, C.byref(n), 1, excl)
    hits = capi.np_from_ptr(hp, n.value, HIT_DT).copy()
    names = [(d.contents.seq[i].name, d.contents.seq[i].len) for i in range(d.contents.n_seq)]
    capi.c_free(hp), port.sd_destroy(d)
    if excl:
        port.sd_destroy(excl)
    return canon(hits), names


def ours(prod, data, route, regrow=None):
    opt = prod.default_opt()
    ctx = prod.mab_create(0)
    if route.startswith("shard"):
        assert prod.mab_shard_init(ctx, 0, 1, None) == 0
    if route == "stream":
        assert prod.mab_load_ingest_text(ctx, data, len(data), opt.min_span, opt.min_match, 1) == 0
    elif route == "shard_stream":
        assert prod.mab_load_ingest_text_sharded(ctx, data, len(data), opt.min_span, opt.min_match, 1) == 0
    else:
        assert prod.mab_load_paf_text(ctx, data, len(data)) == 0
        if route == "ingest":
            prod.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
        elif route == "nocont":
            prod.mab_ingest_nocont(ctx, opt.min_span, opt.min_match, 1, opt.max_hang, opt.int_frac)
        else:
            prod.mab_ingest_sharded(ctx, opt.min_span, opt.min_match, 1)
    n = C.c_size_t(0)
    hp = prod.mab_export_hits(ctx, C.byref(n))
    hits = capi.np_from_ptr(hp, n.value, HIT_DT).copy()
    capi.c_free(hp)
    d = prod.mab_export_dict(ctx)
    names = [(d.contents.seq[i].name, d.contents.seq[i].len) for i in range(d.contents.n_seq)]
    prod.sd_destroy(d)
    st = prod.mab_stats(ctx).contents
    counters = (st.n_lines, st.n_hits_stored, st.n_seq_in)
    if regrow is not None:                  # how often the ingest built a read-name table again
        regrow[route] = st.n_name_regrow
    prod.mab_destroy(ctx)
    return canon(hits), names, counters


def check(prod, port, data, path, routes=ROUTES, regrow=None):
    with open(path, "wb") as f:
        f.write(data)
    want = {False: oracle(port, path, False)}
    n_parsed = parsed_lines(data)
    for route in routes:
        nocont = route == "nocont"
        if nocont not in want:
            want[nocont] = oracle(port, path, True)
        w_hits, w_names = want[nocont]
        hits, names, counters = ours(prod, data, route, regrow)
        assert names == w_names, f"{route}: read names / lengths differ"
        assert np.array_equal(hits, w_hits), f"{route}: hits differ ({len(hits)} vs {len(w_hits)})"
        assert counters == (n_parsed, len(w_hits), len(w_names)), f"{route}: counters {counters}"


def test_tile_and_chunk_boundaries(prod, port, tmp_path):
    data = boundary_text()
    assert len(data) > 3 * CHUNK + TILE
    check(prod, port, data, str(tmp_path / "boundaries.paf"))


@pytest.mark.parametrize("name", list(small_texts()))
def test_small_texts(name, prod, port, tmp_path):
    check(prod, port, small_texts()[name], str(tmp_path / f"{name}.paf"))


def test_line_longer_than_a_chunk(prod, port, tmp_path):
    check(prod, port, chunk_line_text(), str(tmp_path / "giant_line.paf"))


def test_dictionary_overflow(prod, port, tmp_path):
    check(prod, port, overflow_text(), str(tmp_path / "many_names.paf"), routes=["ingest", "stream", "shard"])
