"""BASELINE.json's synthetic configurations at FULL size against the unmodified reference: the reference's GFA for the
same generated PAF was digested once where the reference was built (tests/golden/make_golden_configs.py ->
tests/golden/configs.json); here the PAF is regenerated in memory (same generator, its sha256 is checked too), runs
through the fused CUDA path, and the GFA must have the reference's sha256 -- bit-exact, not "modulo order".

config 2 = 100 K reads / 5 M overlaps, config 3 = 1 M reads / 50 M overlaps (the bench workload), config 4 = 4 M reads /
200 M overlaps (the largest that one 80 GB H100 holds: 12 GB of PAF text and its hits, arcs and sort buffers)."""
import ctypes as C
import hashlib
import json
import os

import pytest

import bench
from miniasm_b200 import capi

pytestmark = pytest.mark.gpu

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "configs.json")))
CASES = [("c2_100k", 100_000, 2), ("c3_1m", 1_000_000, 3), ("c4_4m", 4_000_000, 4)]


@pytest.mark.parametrize("mode", ["plain", "stream"])
@pytest.mark.parametrize("name,n_reads,seed", CASES)
def test_full_size_config_matches_reference_digest(name, n_reads, seed, mode, built):
    if name not in GOLD:
        pytest.skip(f"no golden digest for {name}")
    gold = GOLD[name]
    lib = capi.load_product()
    lib.set_verbose(0)
    buf, n_bytes, n_lines, free = bench.generate(n_reads, seed)
    try:
        assert n_bytes == gold["paf_bytes"]
        view = (C.c_char * n_bytes).from_address(buf.value)
        assert hashlib.sha256(view).hexdigest() == gold["paf_sha256"], "generator output changed: regenerate tests/golden/configs.json"
        del view
        ctx = lib.mab_create(0)
        opt = lib.default_opt()
        if mode == "stream":                                    # load + ingest overlapped, chunk by chunk (pageable source here)
            assert lib.mab_load_ingest_text(ctx, buf, n_bytes, opt.min_span, opt.min_match, 1) == 0
        else:
            assert lib.mab_load_paf_text(ctx, buf, n_bytes) == 0
            lib.mab_ingest(ctx, opt.min_span, opt.min_match, 1) # (synchronises: the host text is no longer needed)
    finally:
        free()
    lib.mab_select(ctx, C.byref(opt), 0, 0, 100)
    lib.mab_layout(ctx, C.byref(opt), 100)
    lib.mab_unitigs(ctx)
    st = lib.mab_stats(ctx).contents
    d, sub, ug = lib.mab_export_dict(ctx), lib.mab_export_sub(ctx), lib.mab_export_ug(ctx)
    gfa = lib.print_to_string("ma_ug_print", ug, d, sub)
    lib.ma_ug_destroy(ug), capi.c_free(sub), lib.sd_destroy(d), lib.mab_destroy(ctx)
    assert len(gfa) == gold["gfa_bytes"]
    assert hashlib.sha256(gfa).hexdigest() == gold["gfa_sha256"]
    reduced = [c for c in gold["stderr_counts"] if c.startswith("asg_arc_del_trans")]
    assert reduced and reduced[0].endswith(f"transitively reduced {st.n_reduced} arcs")
