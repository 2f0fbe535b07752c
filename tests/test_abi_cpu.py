"""CPU tier: the C-ABI library loads without a GPU, exports every symbol include/miniasm_b200.h declares, keeps
the reference's struct layouts, and refuses to compute without a CUDA device (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap

import pytest

from miniasm_b200 import capi

HEADER = os.path.join(capi.ROOT, "include", "miniasm_b200.h")


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = re.findall(r"^[A-Za-z_][A-Za-z0-9_ \*]*?\b([a-z][a-z0-9_]+)\s*\([^;{}]*\)\s*;", src, flags=re.M)
    return sorted(set(names))


def test_every_declared_symbol_is_exported(built):
    dll = C.CDLL(capi.PRODUCT_SO)
    fns = declared_functions()
    assert len(fns) > 60
    missing = [f for f in fns if not hasattr(dll, f)]
    assert not missing, missing
    assert C.c_int.in_dll(dll, "ma_verbose").value == 3


def test_struct_layouts_match_ctypes_and_reference(built, tmp_path, gold):
    """sizeof/offsetof as gcc sees the public header == the ctypes mirrors == the reference's miniasm.h (stored digest of what
    the same program prints with it, tests/refgold.py)."""
    prog = textwrap.dedent("""
        #include <stddef.h>
        #include <stdio.h>
        #include HDR
        int main(void) {
            printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(ma_hit_t), sizeof(ma_sub_t), sizeof(asg_arc_t), sizeof(asg_t), sizeof(ma_utg_t),
                   sizeof(ma_ug_t), sizeof(ma_opt_t), sizeof(sdict_t), sizeof(sd_seq_t));
            printf("%zu %zu %zu %zu %zu\\n", offsetof(asg_t, arc), offsetof(asg_t, seq), offsetof(asg_t, idx), offsetof(ma_utg_t, a), offsetof(ma_ug_t, g));
            return 0;
        }""")
    def layout(k, h):
        c = tmp_path / f"t{k}.c"
        c.write_text(prog.replace("HDR", f'"{h}"'))
        exe = tmp_path / f"t{k}"
        subprocess.check_call(["gcc", "-o", str(exe), str(c)])
        return subprocess.check_output([str(exe)]).decode()

    from oracle import loaders
    outs = [layout(0, HEADER)]
    gold.expect(outs[0], lambda: layout(1, os.path.join(loaders.REFERENCE_SRC, "miniasm.h")))
    sizes = [int(x) for x in outs[0].split()]
    assert sizes[:9] == [32, 8, 16, 40, 40, 32, 56, 24, 16]
    assert sizes[:9] == [capi.HIT_DT.itemsize, capi.SUB_DT.itemsize, capi.ARC_DT.itemsize, C.sizeof(capi.AsgT), C.sizeof(capi.MaUtg),
                         C.sizeof(capi.MaUg), C.sizeof(capi.MaOpt), C.sizeof(capi.Sdict), C.sizeof(capi.SdSeq)]


def _no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


@pytest.mark.skipif(not _no_gpu(), reason="a CUDA device is visible")
@pytest.mark.parametrize("call", ["lib.ma_hit_sub(3, 0.05, 0, 0, None, 4)", "lib.mab_create(0)", "lib.asg_cleanup(lib.asg_init())"])
def test_compute_entry_points_fail_loudly_without_gpu(call, built):
    code = f"import sys; sys.path.insert(0, {capi.ROOT!r})\nfrom miniasm_b200 import capi\nlib = capi.load_product()\n{call}\nprint('survived')"
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode != 0 and "survived" not in r.stdout
    assert "[E::miniasm_b200]" in r.stderr and "no CPU path" in r.stderr


def test_cli_usage_and_version_need_no_gpu(built):
    cli = os.path.join(capi.ROOT, "miniasm_b200", "miniasm-b200")
    r = subprocess.run([cli], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 1 and r.stderr.startswith("Usage: miniasm-b200")
    assert subprocess.run([cli, "-V"], stdout=subprocess.PIPE, text=True).stdout == "0.3-r179\n"
