"""gzip test corpus shared by tests/test_inflate_cpu.py and tests/test_inflate_gpu.py: streams built with Python's zlib over
every compression level, strategy, window size and memory level that changes the block structure, with sync/full flushes,
concatenated members and hand-built headers (FEXTRA with a BGZF subfield, FNAME, FCOMMENT, FHCRC), and a damaged set that a
gzip decoder must reject."""
import random
import struct
import zlib


def deflate_raw(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=15, mem=8, flush_every=0, flush=zlib.Z_SYNC_FLUSH):
    co = zlib.compressobj(level, zlib.DEFLATED, -wbits, mem, strategy)
    if not flush_every:
        return co.compress(data) + co.flush()
    out = []
    for i in range(0, len(data), flush_every):
        out.append(co.compress(data[i:i + flush_every]))
        out.append(co.flush(flush))
    out.append(co.flush())
    return b"".join(out)


def member(data, extra=None, name=None, comment=None, hcrc=False, **kw):
    """One gzip member (RFC 1952) with the optional header fields."""
    flg = (4 if extra is not None else 0) | (8 if name is not None else 0) | (16 if comment is not None else 0) | (2 if hcrc else 0)
    h = bytearray(b"\x1f\x8b\x08" + bytes([flg]) + struct.pack("<I", 0x5f000000) + b"\x00\x03")
    if extra is not None:
        h += struct.pack("<H", len(extra)) + extra
    if name is not None:
        h += name + b"\x00"
    if comment is not None:
        h += comment + b"\x00"
    if hcrc:
        h += struct.pack("<H", zlib.crc32(bytes(h)) & 0xffff)
    return bytes(h) + deflate_raw(data, **kw) + struct.pack("<II", zlib.crc32(data), len(data) & 0xffffffff)


def bgzf(data, block=65280, level=6):
    """BGZF-style: members of at most `block` input bytes, each with a 'BC' extra subfield holding its size - 1."""
    out = []
    for i in range(0, max(len(data), 1), block):
        body = deflate_raw(data[i:i + block], level)
        piece = data[i:i + block]
        hdr_len = 18
        bsize = hdr_len + len(body) + 8 - 1
        extra = b"BC" + struct.pack("<HH", 2, bsize)
        out.append(member(piece, extra=extra, level=level))
    return b"".join(out)


def weird_paf(n=3000, seed=7):
    """PAF lines whose read names hold bytes 0x80-0xFF and control bytes: literals the block-start test does not accept."""
    rnd = random.Random(seed)
    lines = []
    for i in range(n):
        nm = bytes(rnd.choice(list(range(1, 9)) + list(range(0x80, 0x100))) for _ in range(12)) + b"r%d" % i
        tn = b"t%d\x07\x1b" % rnd.randrange(1000)
        lines.append(b"\t".join([nm, b"9000", b"10", b"8000", b"+", tn, b"9500", b"100", b"8100", b"7000", b"8000", b"255"]))
    return b"\n".join(lines) + b"\n"


def valid_corpus(paf):
    """(name, gz bytes, inflated bytes) for a PAF text `paf` (a few hundred KB keeps the CPU tier quick)."""
    small = paf[:60000]
    cases = [("empty", member(b""), b""), ("one_byte", member(b"x"), b"x"), ("one_byte_l0", member(b"\n", level=0), b"\n")]
    for lvl in (0, 1, 6, 9):
        cases.append((f"level{lvl}", member(paf, level=lvl), paf))
    for nm, st in (("filtered", zlib.Z_FILTERED), ("huffman_only", zlib.Z_HUFFMAN_ONLY), ("rle", zlib.Z_RLE), ("fixed", zlib.Z_FIXED)):
        cases.append((nm, member(paf, level=6, strategy=st), paf))
    for wb in range(9, 16):
        cases.append((f"wbits{wb}", member(small, level=6, wbits=wb), small))
    for mem in (1, 9):
        cases.append((f"mem{mem}", member(paf, level=6, mem=mem), paf))
    cases.append(("sync_flush", member(paf, level=1, flush_every=3000), paf))
    cases.append(("full_flush", member(paf, level=6, flush_every=5000, flush=zlib.Z_FULL_FLUSH), paf))
    for k in (2, 7, 50):
        cut = sorted(random.Random(k).sample(range(1, len(paf)), k - 1))
        parts = [paf[a:b] for a, b in zip([0] + cut, cut + [len(paf)])]
        parts.insert(k // 2, b"") # an empty member among them
        cases.append((f"members{k}", b"".join(member(p, level=1 + i % 9) for i, p in enumerate(parts)), paf))
    cases.append(("bgzf", bgzf(paf, block=20000), paf))
    cases.append(("headers", member(paf, extra=b"BC\x02\x00\x00\x00", name=b"reads.paf", comment=b"a comment", hcrc=True, level=1), paf))
    cases.append(("hcrc_only", member(small, hcrc=True), small))
    w = weird_paf()
    cases.append(("weird_names", member(w, level=6), w))
    return cases


def damaged_corpus(paf):
    """(name, gz bytes): streams a decoder must reject."""
    good = member(paf, level=6)
    bad = []
    for k in range(1, 41):
        off = len(good) * k // 41
        bad.append((f"trunc{off}", good[:off]))
    bad.append(("trunc_last_byte", good[:-1]))
    bad.append(("trunc_header", good[:7]))
    flip = bytearray(good)
    flip[len(good) // 2] ^= 0x10
    bad.append(("flipped_bit", bytes(flip)))
    crc = bytearray(good)
    crc[-8] ^= 1
    bad.append(("wrong_crc", bytes(crc)))
    isz = bytearray(good)
    isz[-4] ^= 1
    bad.append(("wrong_isize", bytes(isz)))
    h = bytearray(member(paf, name=b"x.paf", hcrc=True))
    h[h.index(b"x.paf\x00") + 6] ^= 0xff
    bad.append(("bad_fhcrc", bytes(h)))
    bad.append(("trailing_garbage", good + b"garbage\n"))
    bad.append(("trailing_zeros", good + b"\x00" * 16))
    bad.append(("not_gzip", b"\x1f\x8b" + bytes(random.Random(3).randrange(256) for _ in range(5000))))
    bad.append(("bad_method", b"\x1f\x8b\x07" + good[3:]))
    return bad
