"""The fused renderer's residency, from the compiler alone: k_render_fused<OPS = false, ACC16 = true, IN_RANGE = true>, the instantiation
of every default frame without operators, must not spill and must fit all its tiles (one CTA of 128 threads per tile) into the SM's
64K-register file. Its tile count is what lets it hide the gather and wgmma latency, so a register or spill regression that would
silently cost a tile fails here, without a GPU."""
import os
import re
import shutil
import subprocess
import tempfile

from nerfshop_b200 import build

BENCH_KERNEL = "k_render_fusedILb0ELb1ELb1EE"  # k_render_fused<false, true, true>, mangled
REGISTER_FILE = 65536  # 32-bit registers per SM on sm_90


def _compile(tmp: str) -> tuple[str, str]:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    ccbin = ["-ccbin", "/usr/bin/g++"] if os.path.exists("/usr/bin/g++") else []
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", *ccbin, "-Xptxas", "-v", "-keep", "--keep-dir", tmp,
           "-o", os.path.join(tmp, "nsb_kernels.cubin"), os.path.join(build.CSRC, "nsb_kernels.cu")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    ptx = [f for f in os.listdir(tmp) if f.endswith(".ptx")]
    assert len(ptx) == 1, ptx
    with open(os.path.join(tmp, ptx[0])) as fh:
        return res.stdout + res.stderr, fh.read()


def test_bench_instantiation_spills_nothing_and_fits_its_tiles():
    tmp = tempfile.mkdtemp(prefix="nsb_residency_")
    try:
        log, ptx = _compile(tmp)
    finally:
        shutil.rmtree(tmp, True)
    # ptxas -v: "Compiling entry function '<name>'" ... "<n> bytes spill stores" ... "Used <r> registers"
    m = re.search(r"Compiling entry function '(\w*" + BENCH_KERNEL + r"\w*)'.*?(\d+) bytes spill stores.*?Used (\d+) registers", log, re.S)
    assert m, log[-2000:]
    name, spill_stores, regs = m.group(1), int(m.group(2)), int(m.group(3))
    # the launch bound the kernel was compiled for: 128 threads per tile
    b = re.search(r"\.entry " + name + r"\(.*?\)\s*\.maxntid (\d+), 1, 1", ptx, re.S)
    assert b, "no .maxntid for " + name
    threads = int(b.group(1))
    assert threads % 128 == 0 and threads >= 128, threads
    assert spill_stores == 0, f"{name}: {spill_stores} bytes of spill stores"
    regs_alloc = (regs + 7) // 8 * 8  # registers are allocated per thread in units of 8
    assert threads * regs_alloc <= REGISTER_FILE, f"{threads // 128} tiles x 128 threads x {regs} registers > {REGISTER_FILE}"
