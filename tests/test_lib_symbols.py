"""CPU: the C-ABI library loads and exports every symbol include/selfrecon_b200.h declares."""
import ctypes
import os
import re

from helpers import ROOT


def declared_symbols():
    txt = open(os.path.join(ROOT, "include", "selfrecon_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(sr_[a-z0-9_]+)\s*\(", txt)))


def test_header_declares_expected_groups():
    syms = declared_symbols()
    for must in ("sr_minv3x3_f32", "sr_mc_count", "sr_mc_emit", "sr_interp2x3d_fwd_f32",
                 "sr_grid_sample3d_dbwd_f32", "sr_sdf_forward", "sr_deform_forward",
                 "sr_render_forward", "sr_trace_step", "sr_shade_geometry", "sr_fold_linear"):
        assert must in syms


def test_library_exports_every_declared_symbol():
    from selfreconcode_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "run __graft_entry__.build() first"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, missing


def test_binding_table_matches_header():
    from selfreconcode_b200 import _lib
    assert sorted(_lib.SIGNATURES) == declared_symbols()
    lib = _lib.load()
    assert lib.sr_abi_version() == 1
    assert b"sm_90a" in lib.sr_build_info()


def test_struct_layouts_match_c():
    """sizeof of the ctypes mirrors equals what the C compiler lays out (checked with gcc)."""
    import subprocess
    import tempfile
    from selfreconcode_b200 import _lib
    src = '#include <stdio.h>\n#include "selfrecon_b200.h"\nint main(){printf("%zu %zu %zu %zu\\n",' \
          'sizeof(sr_mlp_layer),sizeof(sr_mlp_desc),sizeof(sr_lbs_params),sizeof(sr_trace_params));}'
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        sizes = [int(x) for x in subprocess.check_output([exe]).split()]
    assert sizes == [ctypes.sizeof(_lib.MlpLayer), ctypes.sizeof(_lib.MlpDesc),
                     ctypes.sizeof(_lib.LbsParams), ctypes.sizeof(_lib.TraceParams)]


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "selfreconcode_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), (dp, f)
                assert "liboracle" not in txt, (dp, f)
