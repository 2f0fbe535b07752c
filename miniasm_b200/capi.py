"""ctypes view of the miniasm C ABI (include/miniasm_b200.h).

``load_product()`` -> ``miniasm_b200/libminiasm_b200.so`` (CUDA, sm_90a).  ``Lib`` works for any library that exports the
reference's C API, which is how the test oracles are driven too -- but their loaders live in ``oracle/loaders.py``, not here.
"""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRODUCT_SO = os.path.join(ROOT, "miniasm_b200", "libminiasm_b200.so")

HIT_DT = np.dtype([("qns", "<u8"), ("qe", "<u4"), ("tn", "<u4"), ("ts", "<u4"), ("te", "<u4"),
                   ("ml_rev", "<u4"), ("bl_del", "<u4")])          # ma_hit_t, miniasm.h:29-34
SUB_DT = np.dtype([("s_del", "<u4"), ("e", "<u4")])                   # ma_sub_t, miniasm.h:38-40
ARC_DT = np.dtype([("ul", "<u8"), ("v", "<u4"), ("ol_del", "<u4")])   # asg_arc_t, asg.h:7-11
assert HIT_DT.itemsize == 32 and SUB_DT.itemsize == 8 and ARC_DT.itemsize == 16
DEL = np.uint32(0x80000000)


class MaOpt(C.Structure):                                             # ma_opt_t, miniasm.h:12-27
    _fields_ = [("min_span", C.c_int), ("min_match", C.c_int), ("min_dp", C.c_int), ("min_iden", C.c_float),
                ("max_hang", C.c_int), ("min_ovlp", C.c_int), ("int_frac", C.c_float),
                ("gap_fuzz", C.c_int), ("n_rounds", C.c_int), ("bub_dist", C.c_int), ("max_ext", C.c_int),
                ("min_ovlp_drop_ratio", C.c_float), ("max_ovlp_drop_ratio", C.c_float),
                ("final_ovlp_drop_ratio", C.c_float)]


class SdSeq(C.Structure):                                             # sd_seq_t, sdict.h:6-9
    _fields_ = [("name", C.c_char_p), ("len", C.c_uint32), ("aux_del", C.c_uint32)]


class Sdict(C.Structure):                                             # sdict_t, sdict.h:11-15
    _fields_ = [("n_seq", C.c_uint32), ("m_seq", C.c_uint32), ("seq", C.POINTER(SdSeq)), ("h", C.c_void_p)]


class AsgT(C.Structure):                                              # asg_t, asg.h:17-23
    _fields_ = [("m_arc", C.c_uint32), ("n_arc_srt", C.c_uint32), ("arc", C.c_void_p),
                ("m_seq", C.c_uint32), ("n_seq_symm", C.c_uint32), ("seq", C.c_void_p), ("idx", C.c_void_p)]


class MaUtg(C.Structure):                                             # ma_utg_t, miniasm.h:42-48
    _fields_ = [("len_circ", C.c_uint32), ("start", C.c_uint32), ("end", C.c_uint32), ("m", C.c_uint32),
                ("n", C.c_uint32), ("a", C.POINTER(C.c_uint64)), ("s", C.c_char_p)]


class MaUg(C.Structure):                                              # ma_ug_t, miniasm.h:52-55
    _fields_ = [("n", C.c_size_t), ("m", C.c_size_t), ("a", C.POINTER(MaUtg)), ("g", C.POINTER(AsgT))]


assert C.sizeof(AsgT) == 40 and C.sizeof(MaUtg) == 40 and C.sizeof(MaOpt) == 56

_libc = C.CDLL(None)
_libc.malloc.restype = C.c_void_p
_libc.malloc.argtypes = [C.c_size_t]
_libc.calloc.restype = C.c_void_p
_libc.calloc.argtypes = [C.c_size_t, C.c_size_t]
_libc.free.argtypes = [C.c_void_p]
_libc.fflush.argtypes = [C.c_void_p]
_libc.fopen.restype = C.c_void_p
_libc.fopen.argtypes = [C.c_char_p, C.c_char_p]
_libc.fclose.argtypes = [C.c_void_p]


def c_malloc_copy(arr):
    """malloc'd copy of a numpy array (the C side may realloc/free it)."""
    arr = np.ascontiguousarray(arr)
    p = _libc.malloc(max(arr.nbytes, 16))
    if arr.nbytes:
        C.memmove(p, arr.ctypes.data, arr.nbytes)
    return p


def c_free(p):
    _libc.free(p)


def np_from_ptr(p, n, dtype):
    """Copy n records of dtype out of C memory."""
    dtype = np.dtype(dtype)
    out = np.empty(n, dtype=dtype)
    if n:
        C.memmove(out.ctypes.data, p, n * dtype.itemsize)
    return out


_SIGS = {
    # name: (restype, argtypes)
    "ma_opt_init": (None, [C.POINTER(MaOpt)]),
    "sd_init": (C.POINTER(Sdict), []),
    "sd_destroy": (None, [C.POINTER(Sdict)]),
    "sd_put": (C.c_int32, [C.POINTER(Sdict), C.c_char_p, C.c_uint32]),
    "sd_get": (C.c_int32, [C.POINTER(Sdict), C.c_char_p]),
    "sd_squeeze": (C.c_void_p, [C.POINTER(Sdict)]),
    "ma_hit_no_cont": (C.POINTER(Sdict), [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_float]),
    "ma_hit_read": (C.c_void_p, [C.c_char_p, C.c_int, C.c_int, C.POINTER(Sdict), C.POINTER(C.c_size_t), C.c_int, C.POINTER(Sdict)]),
    "ma_hit_sub": (C.c_void_p, [C.c_int, C.c_float, C.c_int, C.c_size_t, C.c_void_p, C.c_size_t]),
    "ma_hit_cut": (C.c_size_t, [C.c_void_p, C.c_int, C.c_size_t, C.c_void_p]),
    "ma_hit_flt": (C.c_size_t, [C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_void_p, C.POINTER(C.c_float)]),
    "ma_sub_merge": (None, [C.c_size_t, C.c_void_p, C.c_void_p]),
    "ma_hit_contained": (C.c_size_t, [C.POINTER(MaOpt), C.POINTER(Sdict), C.c_void_p, C.c_size_t, C.c_void_p]),
    "ma_sg_gen": (C.POINTER(AsgT), [C.POINTER(MaOpt), C.POINTER(Sdict), C.c_void_p, C.c_size_t, C.c_void_p]),
    "asg_init": (C.POINTER(AsgT), []),
    "asg_destroy": (None, [C.POINTER(AsgT)]),
    "asg_seq_set": (None, [C.POINTER(AsgT), C.c_int, C.c_int, C.c_int]),
    "asg_arc_sort": (None, [C.POINTER(AsgT)]),
    "asg_arc_index": (None, [C.POINTER(AsgT)]),
    "asg_arc_rm": (None, [C.POINTER(AsgT)]),
    "asg_cleanup": (None, [C.POINTER(AsgT)]),
    "asg_symm": (None, [C.POINTER(AsgT)]),
    "asg_arc_del_multi": (C.c_int, [C.POINTER(AsgT)]),
    "asg_arc_del_asymm": (C.c_int, [C.POINTER(AsgT)]),
    "asg_arc_del_trans": (C.c_int, [C.POINTER(AsgT), C.c_int]),
    "asg_arc_del_short": (C.c_int, [C.POINTER(AsgT), C.c_float]),
    "asg_cut_tip": (C.c_int, [C.POINTER(AsgT), C.c_int]),
    "asg_cut_internal": (C.c_int, [C.POINTER(AsgT), C.c_int]),
    "asg_cut_biloop": (C.c_int, [C.POINTER(AsgT), C.c_int]),
    "asg_pop_bubble": (C.c_int, [C.POINTER(AsgT), C.c_int]),
    "ma_ug_gen": (C.POINTER(MaUg), [C.POINTER(AsgT)]),
    "ma_ug_seq": (C.c_int, [C.POINTER(MaUg), C.POINTER(Sdict), C.c_void_p, C.c_char_p]),
    "ma_ug_print": (None, [C.POINTER(MaUg), C.POINTER(Sdict), C.c_void_p, C.c_void_p]),
    "ma_sg_print": (None, [C.POINTER(AsgT), C.POINTER(Sdict), C.c_void_p, C.c_void_p]),
    "ma_ug_destroy": (None, [C.POINTER(MaUg)]),
}

class MabStats(C.Structure):                                          # mab_stats_t
    _fields_ = [(n, C.c_uint64) for n in ("n_lines", "n_hits_stored", "n_seq_in", "n_hits_final", "n_seq_final", "n_arc_sg",
                                          "n_arc_trans_in", "n_reduced", "trans_inner", "n_arc_final", "n_utg")] + \
               [("ms_del_trans_kernel", C.c_double), ("n_kernel_launches", C.c_uint64), ("n_lib_calls", C.c_uint64)] + \
               [(n, C.c_double) for n in ("ms_ingest", "ms_select", "ms_layout", "ms_unitigs")] + \
               [("n_name_regrow", C.c_uint64)]


MAB_READ_FN = C.CFUNCTYPE(C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t)   # mab_text_source_t::read
MAB_REWIND_FN = C.CFUNCTYPE(C.c_int, C.c_void_p)                            # mab_text_source_t::rewind


class MabTextSource(C.Structure):                                     # mab_text_source_t
    _fields_ = [("read", MAB_READ_FN), ("rewind", MAB_REWIND_FN), ("ud", C.c_void_p)]


# symbols include/miniasm_b200.h declares beyond the reference seam
_PRODUCT_ONLY = {
    "mab_create": (C.c_void_p, [C.c_int]),
    "mab_destroy": (None, [C.c_void_p]),
    "mab_stats": (C.POINTER(MabStats), [C.c_void_p]),
    "mab_load_paf_text": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "mab_load_paf_file": (C.c_int, [C.c_void_p, C.c_char_p]),
    "mab_load_paf_gz": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "mab_paf_text": (C.c_size_t, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "mab_ingest": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int]),
    "mab_load_ingest_text": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int]),
    "mab_ingest_windowed": (C.c_int, [C.c_void_p, C.POINTER(MabTextSource), C.c_size_t, C.c_int, C.c_int, C.c_int]),
    "mab_ingest_file_windowed": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_int]),
    "mab_mem_peak": (C.c_size_t, [C.c_void_p, C.c_int]),
    "mab_mem_free": (C.c_size_t, [C.c_void_p]),
    "mab_ingest_nocont": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float]),
    "mab_load_hits": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(Sdict)]),
    "mab_select": (C.c_int, [C.c_void_p, C.POINTER(MaOpt), C.c_int, C.c_int, C.c_int]),
    "mab_layout": (C.c_int, [C.c_void_p, C.POINTER(MaOpt), C.c_int]),
    "mab_unitigs": (C.c_int, [C.c_void_p]),
    "mab_export_dict": (C.POINTER(Sdict), [C.c_void_p]),
    "mab_export_sub": (C.c_void_p, [C.c_void_p]),
    "mab_export_hits": (C.c_void_p, [C.c_void_p, C.POINTER(C.c_size_t)]),
    "mab_export_sg": (C.POINTER(AsgT), [C.c_void_p]),
    "mab_export_ug": (C.POINTER(MaUg), [C.c_void_p]),
    "mab_coverage": (C.c_float, [C.c_void_p]),
    "mab_write_gfa": (C.c_long, [C.c_void_p, C.c_void_p]),
    "mab_write_paf": (C.c_long, [C.c_void_p, C.c_void_p]),
    "mab_write_bed": (C.c_long, [C.c_void_p, C.c_void_p]),
    "mab_write_sg": (C.c_long, [C.c_void_p, C.c_void_p]),
    "mab_reads_prefetch": (C.c_int, [C.c_void_p, C.c_char_p]),
    "mab_write_gfa_reads": (C.c_long, [C.c_void_p, C.c_void_p, C.c_char_p]),
    "mab_event_create": (C.c_void_p, []),
    "mab_event_record": (None, [C.c_void_p, C.c_void_p]),
    "mab_event_elapsed_ms": (C.c_float, [C.c_void_p, C.c_void_p]),
    "mab_event_destroy": (None, [C.c_void_p]),
    "mab_sync": (None, [C.c_void_p]),
    "mab_last_clean": (None, [C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "mab_clean_totals": (None, [C.POINTER(C.c_uint32)] * 4),
    "mab_count_del_trans_inner": (None, [C.c_int]),
    "mab_nccl_unique_id": (C.c_int, [C.c_void_p]),
    "mab_shard_init": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_char_p]),
    "mab_ingest_sharded": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int]),
    "mab_load_ingest_text_sharded": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int]),
    "mab_select_sharded": (C.c_int, [C.c_void_p, C.POINTER(MaOpt)]),
    "mab_layout_sharded": (C.c_int, [C.c_void_p, C.POINTER(MaOpt)]),
    "mab_set_verbose": (None, [C.c_int]),
    "mab_last_del_trans": (None, [C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                  C.POINTER(C.c_uint64), C.POINTER(C.c_double)]),
}


class Lib:
    """A loaded miniasm-ABI library with typed entry points and numpy helpers."""

    def __init__(self, path, product=False, strict=True):
        if not os.path.exists(path):
            raise FileNotFoundError(
                f"{path} is missing: build it first (python -c 'import __graft_entry__ as g; g.build()')")
        self.path = path
        self.dll = C.CDLL(path, mode=os.RTLD_LOCAL | os.RTLD_NOW)
        self.product = product
        sigs = dict(_SIGS)
        if product:
            sigs.update(_PRODUCT_ONLY)
        self.missing = []
        for name, (res, args) in sigs.items():
            try:
                fn = getattr(self.dll, name)
            except AttributeError:
                self.missing.append(name)
                continue
            fn.restype, fn.argtypes = res, args
            setattr(self, name, fn)
        if strict and self.missing:
            raise ImportError(f"{path} lacks symbols: {self.missing}")
        try:
            self._verbose = C.c_int.in_dll(self.dll, "ma_verbose")
        except ValueError:
            self._verbose = None

    # ---- verbosity -----------------------------------------------------------------------------
    def set_verbose(self, level):
        if self._verbose is not None:
            self._verbose.value = level
        if self.product and hasattr(self, "mab_set_verbose"):
            self.mab_set_verbose(level)

    # ---- options -------------------------------------------------------------------------------
    def default_opt(self):
        o = MaOpt()
        self.ma_opt_init(C.byref(o))
        o.min_ovlp = o.min_span                       # main.c:74
        return o

    # ---- graphs --------------------------------------------------------------------------------
    def make_graph(self, arcs, seq, is_srt=False, is_symm=False):
        """Build a host asg_t from numpy arrays (arcs: ARC_DT, seq: uint32 len|del<<31)."""
        g = self.asg_init()
        arcs = np.ascontiguousarray(arcs, dtype=ARC_DT)
        seq = np.ascontiguousarray(seq, dtype=np.uint32)
        g.contents.arc = c_malloc_copy(arcs)
        g.contents.m_arc = max(len(arcs), 1)
        g.contents.n_arc_srt = len(arcs) | (int(is_srt) << 31)
        g.contents.seq = c_malloc_copy(seq)
        g.contents.m_seq = max(len(seq), 1)
        g.contents.n_seq_symm = len(seq) | (int(is_symm) << 31)
        g.contents.idx = None
        return g

    @staticmethod
    def read_graph(g):
        """(arcs, seq, idx or None, is_srt, is_symm) copied out of a host asg_t."""
        c = g.contents
        n_arc, n_seq = c.n_arc_srt & 0x7fffffff, c.n_seq_symm & 0x7fffffff
        arcs = np_from_ptr(c.arc, n_arc, ARC_DT)
        seq = np_from_ptr(c.seq, n_seq, np.uint32)
        idx = np_from_ptr(c.idx, 2 * n_seq, np.uint64) if c.idx else None
        return arcs, seq, idx, bool(c.n_arc_srt >> 31), bool(c.n_seq_symm >> 31)

    def clone_graph(self, g):
        arcs, seq, idx, srt, symm = self.read_graph(g)
        h = self.make_graph(arcs, seq, srt, symm)
        if idx is not None:
            h.contents.idx = c_malloc_copy(idx)
        return h

    # ---- text output through the library's own writers ------------------------------------------
    def print_to_string(self, fn_name, *args):
        import tempfile
        with tempfile.NamedTemporaryFile(delete=False) as tf:
            path = tf.name
        fp = _libc.fopen(path.encode(), b"w")
        getattr(self, fn_name)(*args, fp)
        _libc.fclose(fp)
        with open(path, "rb") as f:
            s = f.read()
        os.unlink(path)
        return s


def load_product(strict=True):
    return Lib(PRODUCT_SO, product=True, strict=strict)

