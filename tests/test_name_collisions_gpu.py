"""Read names built to collide in the read-name dictionaries (tests/golden/name_collisions.json.gz), on every route that names
reads: the ingest's open-addressing dictionary (tab_insert, the windowed win_insert / win_find, the sharded local and global
tables) and the -f name table (ugseq_dev.cu RTab).

Two renamed pafgen sets keep their overlaps and assembly and change only the names:
  pairs    names equal in their hash fragment and their home slot at 2^20 slots, so that the second one to arrive meets the
           first one's slot and has to compare bytes with its witness: in one tile on adjacent lines, in different tiles and
           64 KB windows, both on a tile's last line that ends past the staged overhang (names read from global memory),
           first seen as a target, one dropped by -R;
  cluster  30 000 names homed in 8 192 slots: every probe run is thousands of slots long, holds about a thousand
           fragment-equal groups, wraps past the table's end, overflows the first dictionary (which grows x4) and the
           sharded global table at seed 0 (which is re-seeded).  test_name_collisions_cpu.py proves both from a model.
Expectations come from the oracle port (its own dictionary: 32-bit FNV and strcmp) and the reference's digests."""
import ctypes as C
import gzip
import json
import os
import subprocess

import numpy as np
import pytest

from miniasm_b200 import capi, synth
from miniasm_b200.pipeline import Pipeline
from tests import test_ingest_onepass_gpu as onepass
from tests import test_ingest_windowed_gpu as windowed
from tests.refgold import RECORD
from tests.test_cli_gpu import OURS, REF, outcome

pytestmark = pytest.mark.gpu
product_only = pytest.mark.skipif(RECORD, reason="runs the CUDA library only")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with gzip.open(os.path.join(ROOT, "tests", "golden", "name_collisions.json.gz"), "rb") as _f:
    FX = json.load(_f)
TILE, OVER, KB, MB = 8192, 1024, 1 << 10, 1 << 20     # PT_TILE, PT_OVER: a tile is staged with OVER bytes after it
MIN_SPAN, MIN_MATCH = 2000, 100                        # the default store filter (hit.c:85)
LONG_TAG = b"\tzz:Z:"                                   # an optional field: the port and the reference ignore it
SETS = {"pairs": "-n 4000 -l 2000 -L 30000 -c 30 -j 100 -s 41",      # read lengths over a factor of 15: -R drops hundreds
        "cluster": "-n 30000 -l 3000 -L 3000 -c 25 -s 61"}            # fixed-length reads: ~27 800 survive the selection
ROUTES = onepass.ROUTES


def lines_of(data):
    return data.split(b"\n")[:-1] if data.endswith(b"\n") else data.split(b"\n")


def first_seen(data):
    """name -> (line, role 0 query / 1 target, byte offset of the line) of its first appearance, and the line starts"""
    out, starts, pos = {}, [], 0
    for i, ln in enumerate(lines_of(data)):
        starts.append(pos)
        c = ln.split(b"\t", 6)
        for role, nm in ((0, c[0]), (1, c[5] if len(c) > 5 else None)):
            if nm is not None and nm not in out:
                out[nm] = (i, role, pos)
        pos += len(ln) + 1
    starts.append(pos)
    return out, starts


def tile_of(off):                     # the tile whose '\n' ends the line before (k_parse_tiles)
    return 0 if off == 0 else (off - 1) // TILE


def rename(data, ren):
    out = []
    for ln in lines_of(data):
        c = ln.split(b"\t")
        c[0] = ren.get(c[0], c[0])
        if len(c) > 5:
            c[5] = ren.get(c[5], c[5])
        out.append(b"\t".join(c))
    return b"\n".join(out) + b"\n"


def dropped_by_R(port, path):
    opt = port.default_opt()
    d = port.ma_hit_no_cont(path.encode(), opt.min_span, opt.min_match, opt.max_hang, opt.int_frac)
    names = {d.contents.seq[i].name for i in range(d.contents.n_seq)}
    port.sd_destroy(d)
    return names


def place_pairs(data, dropped):
    """which reads take the pairs' names; roles -> (name a, name b)"""
    fs, starts = first_seen(data)
    order = sorted(fs, key=lambda n: 2 * fs[n][0] + fs[n][1])
    by_line = {}
    for n in order:
        by_line.setdefault(fs[n][0], []).append(n)
    kind = {k: [p for p in FX["pairs"] if p["kind"] == k] for k in ("prefix", "length", "short")}
    head = [kind["prefix"][0], kind["length"][0], kind["short"][0], kind["length"][1]]
    pairs = head + [p for p in FX["pairs"] if p not in head and p is not kind["prefix"][1]] + [kind["prefix"][1]]  # in the order of the roles
    ren, roles, used = {}, {}, set()

    def take(role, x, y):
        p = pairs[len(roles)]
        ren[x], ren[y] = p["a"].encode(), p["b"].encode()
        used.update((x, y))
        roles[role] = (p["a"].encode(), p["b"].encode())

    def first(pred):
        return next(n for n in order if n not in used and pred(n, *fs[n]))

    # both first seen in tile 0, on adjacent lines (tile-staged witness, same 64 KB window)
    x = first(lambda n, ln, r, off: ln > 0 and ln + 1 in by_line and starts[ln + 2] + 128 < TILE)
    take("same_tile", x, by_line[fs[x][0] + 1][0])
    # first seen in tile 0 and at 256 KB and after: different tiles, and 64 KB windows 0 and >= 3 (witness in the name store)
    take("windows", first(lambda n, ln, r, off: off + 2 * KB < TILE), first(lambda n, ln, r, off: off >= 256 * KB))
    # first seen as a target
    x = first(lambda n, ln, r, off: off >= 400 * KB and r == 1)
    take("target", x, first(lambda n, ln, r, off: off > fs[x][2] + 10 * KB))
    # one of the two is dropped by -R
    x = first(lambda n, ln, r, off: off >= 500 * KB and n in dropped)
    take("dropped", x, first(lambda n, ln, r, off: off > fs[x][2] and n not in dropped))
    rest = [n for n in order if n not in used]
    step = len(rest) // (2 * (len(pairs) - len(roles)) + 1)
    k = 0
    while len(roles) < len(pairs) - 1:
        take(f"spread{k}", rest[(2 * k + 1) * step], rest[(2 * k + 2) * step])
        k += 1
    # query and target of one stored line, both first seen at 300 KB or later (so nothing before 300 KB moves); lengthen_line then
    # makes that line end past the tile's staged overhang, so the parse reads both names from global memory
    lines = lines_of(data)

    def fits(n, ln, r, off):
        c = lines[ln].split(b"\t")
        y = c[5]
        return (off >= 300 * KB and r == 0 and y != n and y not in used and fs[y][2] >= 300 * KB and
                int(c[3]) - int(c[2]) >= MIN_SPAN and int(c[8]) - int(c[7]) >= MIN_SPAN and int(c[9]) >= MIN_MATCH)
    x = first(fits)
    take("tile_last", x, lines[fs[x][0]].split(b"\t")[5])
    return ren, roles


def lengthen_line(data, q, t):
    """the line with query q and target t gets an optional field that makes it end PT_OVER + 512 bytes past its tile: it is the
    tile's last line and ends beyond the staged bytes (k_parse_tiles parses it, and enters its names, from global memory)"""
    lines, pos = lines_of(data), 0
    for i, ln in enumerate(lines):
        c = ln.split(b"\t", 6)
        if c[0] == q and c[5] == t:
            pad = (tile_of(pos) + 1) * TILE + OVER + 512 - (pos + len(ln)) - len(LONG_TAG)
            assert pad > 0
            lines[i] = ln + LONG_TAG + b"A" * pad
            return b"\n".join(lines) + b"\n"
        pos += len(ln) + 1
    raise AssertionError("no such line")


@pytest.fixture(scope="module")
def sets(built, port, paf_dir):
    out = {}
    for name, args in SETS.items():
        src = synth.generate(args, os.path.join(paf_dir, f"nc_{name}_src.paf"))
        data = open(src, "rb").read()
        if name == "pairs":
            ren, roles = place_pairs(data, dropped_by_R(port, src))
        else:
            fs, _ = first_seen(data)
            order = sorted(fs, key=lambda n: 2 * fs[n][0] + fs[n][1])
            assert len(order) <= len(FX["cluster"])
            ren, roles = {n: FX["cluster"][k].encode() for k, n in enumerate(order)}, None
        data = rename(data, ren)
        if roles:
            data = lengthen_line(data, *roles["tile_last"])
        assert len(data) // 24 + 1024 <= 8 << 20              # the first dictionary has 2^20 slots (tab_cap_for)
        path = os.path.join(paf_dir, f"nc_{name}.paf")
        with open(path, "wb") as f:
            f.write(data)
        out[name] = (path, data, roles)
    return out


def test_pairs_sit_where_they_should(sets, port):
    path, data, roles = sets["pairs"]
    fs, starts = first_seen(data)
    a, b = roles["same_tile"]
    assert fs[b][0] == fs[a][0] + 1 and tile_of(fs[a][2]) == tile_of(fs[b][2]) == 0 and fs[b][2] < 60 * KB
    a, b = roles["windows"]
    assert fs[a][2] < 60 * KB and fs[b][2] >= 128 * KB and tile_of(fs[a][2]) != tile_of(fs[b][2])
    a, b = roles["tile_last"]
    ln = fs[a][0]
    c = lines_of(data)[ln].split(b"\t")
    assert fs[a][1] == 0 and c[0] == a and c[5] == b and int(c[3]) - int(c[2]) >= MIN_SPAN   # a first seen there, with b
    eol = starts[ln + 1] - 1                               # its '\n': past the tile and past the overhang staged with it
    assert eol > (tile_of(fs[a][2]) + 1) * TILE + OVER
    assert 1 in (fs[roles["target"][0]][1], fs[roles["target"][1]][1])
    a, b = roles["dropped"]
    kept = {n for n, _ in onepass.oracle(port, path, True)[1]}
    assert a not in kept and b in kept
    assert all(n in fs for r in roles.values() for n in r) and len(roles) == len(FX["pairs"])


# ---- ingest state: every route against the oracle port -----------------------------------------------------------------------
@product_only
@pytest.mark.parametrize("which", ["pairs", "cluster"])
def test_ingest_routes(which, sets, prod, port, tmp_path):
    path, data, _ = sets[which]
    regrow = {}
    onepass.check(prod, port, data, str(tmp_path / "in.paf"), ROUTES, regrow)
    assert set(regrow) == set(ROUTES)
    if which == "pairs":
        assert all(v == 0 for v in regrow.values()), regrow
    else:   # the first dictionary overflows (probe limit); the sharded global table overflows at seed 0 as well
        assert all(v >= 1 for v in regrow.values()) and regrow["shard"] >= 2 and regrow["shard_stream"] >= 2, regrow


@product_only
@pytest.mark.parametrize("which", ["pairs", "cluster"])
def test_ingest_windowed(which, sets, prod, port, tmp_path):
    path, data, _ = sets[which]
    regrow = {}
    windowed.check(prod, port, data, str(tmp_path / "in.paf"), [64 * KB, MB], regrow)
    assert all((v == 0) if which == "pairs" else (v >= 1) for v in regrow.values()) and len(regrow) == 2, regrow


# ---- the whole pipeline -------------------------------------------------------------------------------------------------------
@product_only
@pytest.mark.parametrize("which", ["pairs", "cluster"])
def test_fused_gfa_equals_port(which, sets, prod, port):
    path, _, _ = sets[which]
    ctx = prod.mab_create(0)
    opt = prod.default_opt()
    assert prod.mab_load_paf_file(ctx, path.encode()) == 0
    prod.mab_ingest(ctx, opt.min_span, opt.min_match, 1)
    prod.mab_select(ctx, C.byref(opt), 0, 0, 100)
    prod.mab_layout(ctx, C.byref(opt), 100)
    prod.mab_unitigs(ctx)
    d, sub, ug = prod.mab_export_dict(ctx), prod.mab_export_sub(ctx), prod.mab_export_ug(ctx)
    gfa = prod.print_to_string("ma_ug_print", ug, d, sub)
    st = prod.mab_stats(ctx).contents
    n_final = st.n_seq_final
    prod.ma_ug_destroy(ug), capi.c_free(sub), prod.sd_destroy(d), prod.mab_destroy(ctx)
    assert gfa == Pipeline(port, path).run_all()
    assert gfa.startswith(b"S\t")
    if which == "cluster":             # the -f table of the layout then has 2^16 slots, the mask the foreign names are homed under
        assert 16384 < n_final <= 32768, n_final


def cli(args, env=None):
    r = subprocess.run([OURS] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=dict(os.environ, **(env or {})))
    return r.returncode, r.stdout, r.stderr


def same(gold, args, env=None):
    rc, out, err = cli(args, env)
    assert rc == 0, err.decode()[-2000:]
    gold.cli("exact", args, outcome(rc, out), lambda: outcome(*_ref(args)))
    return out


def _ref(args):
    r = subprocess.run([REF] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    return r.returncode, r.stdout


@pytest.mark.parametrize("which", ["pairs", "cluster"])
@pytest.mark.parametrize("opts,env", [([], None), (["-S", "2", "-p", "bed"], None), (["-R"], None),
                                      ([], {"MINIASM_B200_INGEST": "windowed", "MINIASM_B200_WINDOW": "65536"})],
                         ids=["default", "S2_bed", "R", "windowed"])
def test_cli_against_the_reference(which, opts, env, sets, gold):
    path, _, _ = sets[which]
    out = same(gold, opts + [path], env)
    assert out


# ---- -f: record lookups along the cluster's chain -----------------------------------------------------------------------------
def _lengths(data):
    lens = {}
    for ln in lines_of(data):
        c = ln.split(b"\t")
        lens.setdefault(c[0], int(c[1]))
        lens.setdefault(c[5], int(c[6]))
    return lens


def write_reads(data, path, fq):
    """records for the layout reads (every 40th has none), a later record of every 9th with other bases (it wins), and the foreign
    names as records of no read; only A/C/G/T, so an N in a read's piece means a record that was not found"""
    rng = np.random.default_rng(5)
    lens = _lengths(data)
    names = sorted(lens)
    rng.shuffle(names)
    pool = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 1 << 22)].tobytes()
    missing = set(names[::40])
    with open(path, "wb") as f:
        def rec(nm, n):
            o = int(rng.integers(0, len(pool) - n))
            s = pool[o:o + n]
            if fq:
                f.write(b"@" + nm + b"\n" + s + b"\n+\n" + b"I" * n + b"\n")
            else:
                f.write(b">" + nm + b" x\n" + b"\n".join(s[i:i + 80] for i in range(0, n, 80)) + b"\n")
        foreign = [n.encode() for n in FX["foreign"]]
        for k, nm in enumerate(names):
            if k % 100 == 0 and foreign:
                for g in foreign[:3]:
                    rec(g, 500)
                foreign = foreign[3:]
            if nm in missing:
                continue
            rec(nm, lens[nm])
            if k % 9 == 0:
                rec(nm, lens[nm])
        for g in foreign:
            rec(g, 500)
    return missing


def pieces_with_n(gfa, missing):
    """(unitig, read) of the a-lines whose piece of the S line holds an N although the read has a record"""
    seq, bad = {}, []
    for ln in gfa.split(b"\n"):
        c = ln.split(b"\t")
        if c[0] == b"S":
            seq[c[1]] = c[2]
        elif c[0] == b"a":
            rd = c[3].rsplit(b":", 1)[0]
            off, n = int(c[2]), int(c[5])
            if rd not in missing and b"N" in seq[c[1]][off:off + n]:
                bad.append((c[1], rd))
    return bad


@pytest.mark.parametrize("fq", [False, True], ids=["fasta", "fastq4"])
def test_reads_on_one_long_chain(fq, sets, tmp_path, gold):
    path, data, _ = sets["cluster"]
    reads = str(tmp_path / ("nc_cluster_reads." + ("fq" if fq else "fa")))
    missing = write_reads(data, reads, fq)
    out = same(gold, ["-f", reads, path])
    if not RECORD:
        rc, host, err = cli(["-f", reads, path], {"MAB_GPU_SEQ": "0"})
        assert rc == 0 and host == out, err.decode()[-2000:]
    assert not pieces_with_n(out, missing)
    assert b"N" in out                                 # the reads without a record do leave N's


def n_gpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@product_only
@pytest.mark.skipif(n_gpus() < 2, reason="needs at least 2 GPUs")
@pytest.mark.parametrize("which", ["pairs", "cluster"])
def test_two_gpus(which, sets):
    path, _, _ = sets[which]
    rc1, one, err1 = cli([path])
    rc2, two, err2 = cli([path], {"MINIASM_B200_GPUS": "2"})
    assert rc1 == 0 and rc2 == 0, err2.decode()[-2000:]
    assert two == one
