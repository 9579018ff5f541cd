"""CPU tests of the drop-in boundary: the C-ABI library builds for sm_90a, loads, and exports exactly
the symbols include/nerfshop_b200.h declares (no compute calls: there is no GPU in CI)."""
import ctypes as C
import os
import re

import numpy as np

from nerfshop_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "nerfshop_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(nsb_[a-z0-9_]+)\s*\(", src)))


def test_header_and_bindings_agree():
    assert _declared_symbols() == sorted(abi.EXPORTED_SYMBOLS)


def test_library_exports_every_declared_symbol(built_lib):
    lib = C.CDLL(built_lib)
    for name in _declared_symbols():
        assert hasattr(lib, name), name
    lib.nsb_abi_version.restype = C.c_int
    assert lib.nsb_abi_version() == abi.NSB_ABI_VERSION


def test_struct_layouts_match_the_c_compiler(tmp_path):
    """sizeof/offsetof of the ABI structs as gcc sees them == the ctypes mirrors."""
    import subprocess

    prog = tmp_path / "sz.c"
    prog.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "nerfshop_b200.h"\n'
        "int main(){printf(\"%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n\", sizeof(NsbModelDesc), sizeof(NsbFrame), sizeof(NsbEditOp), sizeof(NsbAffineBox),"
        " sizeof(NsbRenderStats), offsetof(NsbFrame, tile_rank), offsetof(NsbEditOp, selection_box), offsetof(NsbEditOp, tet_lut_offsets),"
        " sizeof(NsbGridUpdate), offsetof(NsbGridUpdate, rng_state), offsetof(NsbGridUpdate, apply_operators), sizeof(NsbBoundarySampling),"
        " offsetof(NsbBoundarySampling, seed), sizeof(NsbTonemap));return 0;}\n"
    )
    exe = tmp_path / "sz"
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [C.sizeof(abi.NsbModelDesc), C.sizeof(abi.NsbFrame), C.sizeof(abi.NsbEditOp), C.sizeof(abi.NsbAffineBox), C.sizeof(abi.NsbRenderStats),
            abi.NsbFrame.tile_rank.offset, abi.NsbEditOp.selection_box.offset, abi.NsbEditOp.tet_lut_offsets.offset,
            C.sizeof(abi.NsbGridUpdate), abi.NsbGridUpdate.rng_state.offset, abi.NsbGridUpdate.apply_operators.offset, C.sizeof(abi.NsbBoundarySampling),
            abi.NsbBoundarySampling.seed.offset, C.sizeof(abi.NsbTonemap)]
    assert got == want


def test_model_size_query_needs_no_gpu(built_lib):
    from nerfshop_b200 import synthetic as syn

    lib = abi.load_library()
    n = C.c_uint64()
    desc = syn.model_desc(4)
    assert lib.nsb_model_n_params(C.byref(desc), C.byref(n)) == abi.NSB_OK
    assert n.value == 10240 + 13074912
    bad = syn.model_desc(4)
    bad.n_neurons = 128
    assert lib.nsb_model_n_params(C.byref(bad), C.byref(n)) == abi.NSB_ERR_INVALID
    assert b"base.json" in lib.nsb_last_error()


def test_no_cpu_fallback_without_gpu(built_lib):
    """On a box without a GPU context creation fails loudly instead of falling back."""
    import torch

    if torch.cuda.is_available():
        return
    lib = abi.load_library()
    ctx = C.c_void_p()
    assert lib.nsb_create(0, C.byref(ctx)) != abi.NSB_OK
    from nerfshop_b200.renderer import NerfRenderer

    try:
        NerfRenderer(0)
        raise AssertionError("expected NsbError")
    except abi.NsbError:
        pass
