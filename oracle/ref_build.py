"""Builds oracle/_ref/libnerfshop_ref.so: the reference's OWN render-path sources, compiled for the CPU.

TEST INFRASTRUCTURE ONLY. Nothing under nerfshop_b200/ may import or link it (tests/test_product_isolation.py).

What is compiled, from where it lies under /root/reference (never copied into the repository):
  * whole files / headers, included as they are: src/common_nerf.cu, common.h, common_nerf.h, common_device.cuh,
    bounding_box.cuh, triangle.cuh, random_val.cuh, nerf.h, envmap.cuh, editing/tools/{selection_utils.h,
    affine_bounding_box.cuh, mvc.h, svd3.h}, editing/datastructures/{tet_mesh.h, mesh.h};
  * named functions cut out of translation units whose other contents need the absent submodules (GUI, training,
    tiny-cuda-nn internals): see EXTRACTS. They are located by signature, cut by brace matching, written to a scratch
    directory under oracle/_ref/ that is deleted after the compile, and #included by oracle/ref_driver.cpp.
The absent dependencies (Eigen fork, tiny-cuda-nn, tinylogger, json, OpenGL) are replaced by the small stand-ins in
oracle/ref_shim/ (our code, written for this purpose). tiny-cuda-nn's network itself (hash grid + MLPs) is NOT available:
ref_driver.cpp's NerfNetwork calls back into a function pointer supplied by the test (the oracle's encode + MLP).

Compiler flags (GXX_KERNELS): -ffp-contract=fast -mfma, so that gcc contracts a*b+c into FMAs inside expressions the way nvcc's default
-fmad=true does for the reference's device code (CMakeLists.txt:71-80 sets no --fmad=false). The two compilers' contraction
rules are not guaranteed to coincide; tests/test_oracle_vs_ref.py reports every comparison as a count of differing values.

The GPU box has no /root/reference: the .so is built here and travels with the repository snapshot (git-ignored).

Every library of oracle/_ref (this module's two and those of the other oracle/ref_*_build.py) is built by build_library: its cut-outs
(write_cutouts), one of the flag lists below plus its own include directories, and a rebuild whenever a file of dependencies() is newer.
NSB_REF_KEEP_GEN=1 keeps the cut-outs (and nvcc's intermediate files) under oracle/_ref/gen*/ for inspection.
"""
from __future__ import annotations

import os
import re
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("NSB_REFERENCE_ROOT", "/root/reference")
OUT_DIR = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT_DIR, "libnerfshop_ref.so")
LIB_CUDA = os.path.join(OUT_DIR, "libnerfshop_ref_cuda.so")
DRIVER_CUDA = os.path.join(HERE, "ref_driver_cuda.cu")
SHIM = os.path.join(HERE, "ref_shim")
DRIVER = os.path.join(HERE, "ref_driver.cpp")
REF_INCLUDES = ["-I", os.path.join(REF, "include"), "-I", os.path.join(REF, "src")]

_GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
# the compiler and the flags of each kind of build; a library adds its include directories, its driver and what else it names
NVCC = [shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
        "--extended-lambda", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-shared", "-w"] + (
        ["-ccbin", "/usr/bin/g++"] if os.path.exists("/usr/bin/g++") else [])
# the reference's kernels on the CPU: OpenMP over the launch grid, and a*b+c contracted as nvcc's -fmad=true does
GXX_KERNELS = [_GXX, "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=fast", "-mfma", "-fno-fast-math",
               "-Wno-deprecated-declarations", "-Wno-attributes", "-w"]
# the reference's host code: its host build does not contract
GXX_HOST = [_GXX, "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-w"]

# {name: (reference file, [(kind, regex of the first line[, regex of the last line]), ...])}, written to name.inc by write_cutouts; kind
# "fn" = function definition (brace matched, a preceding `template <...>` line is taken along), "stmt" = statement up to the terminating
# ';', "range" = from the first line to the next line that matches the second regex
EXTRACTS = {
    "testbed_nerf": ("src/testbed_nerf.cu", [
        ("stmt", r"^static constexpr uint32_t MARCH_ITER\b"),
        ("stmt", r"^static constexpr uint32_t MIN_STEPS_INBETWEEN_COMPACTION\b"),
        ("stmt", r"^static constexpr uint32_t MAX_STEPS_INBETWEEN_COMPACTION\b"),
        ("fn", r"^__device__ float network_to_rgb_derivative\("),
        ("fn", r"^__device__ float network_to_density_derivative\("),
        ("fn", r"^__global__ void grid_to_bitfield\("),
        ("fn", r"^__global__ void bitfield_max_pool\("),
        ("fn", r"^__global__ void advance_pos_nerf\("),
        ("fn", r"^__global__ void generate_nerf_network_inputs_at_current_position\("),
        ("fn", r"^__global__ void compute_nerf_density\("),
        ("fn", r"^__global__ void generate_next_nerf_network_inputs\("),
        ("fn", r"^__global__ void composite_kernel_nerf\("),
        ("fn", r"^__global__ void shade_kernel_nerf\("),
        ("fn", r"^__global__ void compact_kernel_nerf\("),
        ("fn", r"^__global__ void init_rays_with_payload_kernel_nerf\("),
        ("fn", r"^void Testbed::NerfTracer::init_rays_from_camera\("),
        ("fn", r"^__global__ void clear_empty_space\("),
        # the occupancy update through the operators (SURVEY.md section 8 row (f)-2), CPU build only (ref_common.inl guards the members)
        ("fn", r"^__global__ void splat_grid_samples_nerf_max_nearest_neighbor_already_activated\("),
        ("fn", r"^__global__ void ema_grid_samples_nerf\("),
        ("fn", r"^__global__ void activate_network_density\("),
        ("fn", r"^void Testbed::update_density_grid_nerf_operator\("),
        ("fn", r"^void Testbed::update_density_grid_mean_and_bitfield\("),
        ("fn", r"^uint32_t Testbed::NerfTracer::trace\("),
        ("fn", r"^void Testbed::NerfTracer::enlarge\("),
        ("fn", r"^void Testbed::render_nerf\("),
    ]),
    # frame post-process (SURVEY.md section 8 row (f)-4): accumulate / tonemap
    "render_buffer": ("src/render_buffer.cu", [
        ("fn", r"^__global__ void accumulate_kernel\("),
        ("fn", r"^__device__ Array3f tonemap\(Array3f x, ETonemapCurve curve\)"),
        ("fn", r"^__device__ Array3f tonemap\(Array3f col, const Array3f& exposure"),
        ("fn", r"^__global__ void tonemap_kernel\("),
    ]),
    # the edits I/O glue (SURVEY.md section 8 row (f)-3): Eigen <-> json and BoundingBox <-> json; included by the shadow json_binding.h
    "json_binding": ("include/neural-graphics-primitives/json_binding.h", [
        ("range", r"^namespace Eigen \{", r"^\}$"),
        ("range", r"^NGP_NAMESPACE_BEGIN$", r"^NGP_NAMESPACE_BEGIN$"),
        ("fn", r"^inline void to_json\(nlohmann::json& j, const BoundingBox& box\)"),
        ("fn", r"^inline void from_json\(const nlohmann::json& j, BoundingBox& box\)"),
        ("range", r"^NGP_NAMESPACE_END$", r"^NGP_NAMESPACE_END$"),
    ]),
    "cage_deformation": ("src/editing/cage_deformation.cu", [
        ("fn", r"^__global__ void interpolate_tet_pos\("),
        ("fn", r"^__global__ void interpolate_tet\("),
        ("fn", r"^__global__ void compute_poisson_residual_density_kernel\("),
        ("fn", r"^__global__ void compute_residual_poisson_kernel\("),
    ]),
    "affine_duplication": ("src/editing/affine_duplication.cu", [
        ("fn", r"^__device__ Vector3f warp_direction_ad\("),
        ("fn", r"^__device__ Vector3f unwarp_direction_ad\("),
        ("fn", r"^__global__ void translate_in_box_pos\("),
        ("fn", r"^__global__ void translate_in_box\("),
    ]),
    "tet_mesh": ("src/editing/datastructures/tet_mesh.cu", [
        ("fn", r"^void TetMesh<float_t, point_t>::post_update_vertices\("),
        ("fn", r"^void TetMesh<float_t, point_t>::update_all_indices\("),
        ("fn", r"^void TetMesh<float_t, point_t>::update_local_rotations\("),
        ("fn", r"^void TetMesh<float_t, point_t>::build_original_tet_grid\("),
        ("stmt", r"^static std::vector<std::vector<std::tuple<int, int, int, int>>> up_ids;"),
        ("stmt", r"^static std::vector<int> tet_sums;"),
        ("fn", r"^void TetMesh<float_t, point_t>::build_tet_grid\("),
    ]),
    "cage": ("src/editing/datastructures/cage.cu", [
        ("fn", r"^void Cage<float_t, point_t>::compute_mvc\("),
        ("fn", r"^void Cage<float_t, point_t>::interpolate_with_mvc\(const std::vector<std::vector<float_t>>& weights"),
    ]),
    # the membrane blend (SURVEY.md section 8 row (f)-4): the loop of GrowingSelection::interpolate_poisson_boundary, between the two
    # compute_poisson_boundary calls above it (network evaluation, std::rand) and the uploads below it; ref_driver.cpp supplies the named objects
    "growing_selection": ("src/editing/tools/growing_selection.cu", [
        ("range", r"^\tuint32_t n_tet_vertices = tet_interpolation_mesh->vertices\.size\(\);", r"^\t\tboundary_residual_density_host\[i\] = std::max\(boundary_residual_density_host\[i\], 0\.f\);"),
    ]),
    # the membrane boundary values (row (f)-4): GrowingSelection::compute_poisson_boundary with its two kernels, and project_sh9
    "growing_selection_boundary": ("src/editing/tools/growing_selection.cu", [
        ("fn", r"^__global__ void activate_network_output\("),
        ("fn", r"^__global__ void filter_empty\("),
        ("fn", r"^void GrowingSelection::compute_poisson_boundary\("),
    ]),
    "sh_utils": ("src/editing/tools/sh_utils.cu", [
        ("fn", r"^SH9RGB project_sh9\(const Eigen::Vector3f& dir, const Eigen::Vector3f& rgb"),
    ]),
    "selection_utils": ("src/editing/tools/selection_utils.cu", [
        ("fn", r"^Eigen::Vector3f get_cell_pos\("),
        ("fn", r"^Eigen::Vector3i get_cell_at_pos\("),
    ]),
}


LAUNCH_RX = re.compile(r"(\w+)<<<\s*([^,>]+),\s*([^,>]+)(?:,[^>]*)?>>>\(")


def _strip_for_braces(line: str, in_block: bool):
    """Returns (code without comments/strings, still inside a /* */ block)."""
    out = []
    i = 0
    n = len(line)
    while i < n:
        if in_block:
            j = line.find("*/", i)
            if j < 0:
                return "".join(out), True
            i = j + 2
            in_block = False
            continue
        c = line[i]
        if line.startswith("//", i):
            break
        if line.startswith("/*", i):
            in_block = True
            i += 2
            continue
        if c == '"' or c == "'":
            q = c
            i += 1
            while i < n and line[i] != q:
                i += 2 if line[i] == "\\" else 1
            i += 1
            continue
        out.append(c)
        i += 1
    return "".join(out), in_block


def cut(lines, kind, pattern, last=None):
    """(first, last) index of the lines of one cut-out; its first line is the one line that matches pattern."""
    rx = re.compile(pattern)
    hits = [i for i, l in enumerate(lines) if rx.search(l)]
    if len(hits) != 1:
        raise RuntimeError(f"anchor {pattern!r}: {len(hits)} matches (expected exactly 1)")
    start = hits[0]
    first = start
    if kind == "fn":
        while first > 0 and lines[first - 1].lstrip().startswith("template"):
            first -= 1
        depth = 0
        seen = False
        in_block = False
        i = start
        while True:
            code, in_block = _strip_for_braces(lines[i], in_block)
            for ch in code:
                if ch == "{":
                    depth += 1
                    seen = True
                elif ch == "}":
                    depth -= 1
            if seen and depth == 0:
                break
            i += 1
        end = i
    elif kind == "range":
        # statements out of the middle of a member whose surroundings cannot be compiled here
        rx_last = re.compile(last)
        ends = [i for i in range(start, len(lines)) if rx_last.search(lines[i])]
        if not ends:
            raise RuntimeError(f"anchor {last!r}: no match after line {start + 1}")
        end = ends[0]
    else:
        i = start
        while ";" not in lines[i]:
            i += 1
        end = i
    return first, end


def write_cutouts(table, gen_dir: str, transform=lambda line: line):
    """Writes each entry of a table shaped like EXTRACTS to gen_dir/name.inc: its cut-outs in order, each line passed through transform,
    each behind a #line directive to where it lies in the reference. Returns the manifest lines (file:first-last, anchor)."""
    manifest = []
    for name, (rel, items) in table.items():
        path = os.path.join(REF, rel)
        with open(path, "r", encoding="utf-8", errors="replace") as fh:
            lines = fh.read().split("\n")
        parts = []
        for item in items:
            a, b = cut(lines, *item)
            manifest.append(f"{rel}:{a + 1}-{b + 1}  {item[1]}")
            body = [transform(l) for l in lines[a:b + 1]]
            parts.append(f"// ---- {rel}:{a + 1}-{b + 1} ----\n#line {a + 1} \"{path}\"\n" + "\n".join(body) + "\n")
        with open(os.path.join(gen_dir, name + ".inc"), "w") as fh:
            fh.write("\n".join(parts))
    return manifest


def extract_all(gen_dir: str):
    """EXTRACTS, with the one mechanical rewrite: CUDA's launch syntax is not C++ (same kernel, same arguments, same grid)."""
    return write_cutouts(EXTRACTS, gen_dir, lambda line: LAUNCH_RX.sub(r"nsb_launch(\2, \3, \1, ", line))


def available() -> bool:
    return os.path.isdir(os.path.join(REF, "src")) and os.path.exists(os.path.join(REF, "src", "testbed_nerf.cu"))


_INCLUDE_RX = re.compile(r'^\s*#\s*include\s*"([^"]+)"', re.M)


def dependencies(driver: str, shims, module: str):
    """The repository's files a library is built from: its driver and every file the driver's quoted #includes reach in the repository,
    every file under its stand-in directories, this module and the library's own build module."""
    deps, todo = set(), [os.path.abspath(driver)]
    while todo:
        path = todo.pop()
        if path in deps:
            continue
        deps.add(path)
        with open(path, "r", encoding="utf-8") as fh:
            for inc in _INCLUDE_RX.findall(fh.read()):
                inc = os.path.normpath(os.path.join(os.path.dirname(path), inc))
                if os.path.isfile(inc):
                    todo.append(inc)
    for d in shims:
        for root, _, files in os.walk(d):
            deps.update(os.path.join(root, f) for f in files)
    deps.update((os.path.abspath(__file__), os.path.abspath(module)))
    return sorted(deps)


def stale(lib: str, deps) -> bool:
    return not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps)


def build_library(lib: str, driver: str, gen_name: str, compile_cmd, cut, shims, module: str, force: bool = False):
    """Builds one library of oracle/_ref unless it is newer than every file of dependencies(driver, shims, module): cut(gen) writes the
    cut-outs into the fresh directory oracle/_ref/<gen_name>, compile_cmd(gen) is run, and the cut-outs (reference source) are deleted
    unless NSB_REF_KEEP_GEN=1. Returns the library's path, or None when the reference's sources are absent and no prebuilt library
    exists."""
    if not available():
        return lib if os.path.exists(lib) else None
    if not force and not stale(lib, dependencies(driver, shims, module)):
        return lib
    gen = os.path.join(OUT_DIR, gen_name)
    shutil.rmtree(gen, ignore_errors=True)
    os.makedirs(gen)
    cut(gen)
    cmd = compile_cmd(gen)
    keep = os.environ.get("NSB_REF_KEEP_GEN") == "1"
    if keep and cmd[0] == NVCC[0]:
        cmd += ["--keep", "--keep-dir", gen]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if not keep:
        shutil.rmtree(gen, ignore_errors=True)
    if res.returncode != 0:
        raise RuntimeError(f"oracle/_ref/{os.path.basename(lib)} build failed:\n" + res.stdout + res.stderr[-6000:])
    return lib


def build(force: bool = False, verbose: bool = False):
    """Returns the path of the library, or None when /root/reference is absent (GPU box) and no prebuilt library exists."""
    manifest = []

    def cut_and_record(gen):
        manifest.extend(extract_all(gen))

    lib = build_library(LIB, DRIVER, "gen", lambda gen: GXX_KERNELS + ["-I", SHIM, "-I", gen, *REF_INCLUDES, "-x", "c++", DRIVER, "-o", LIB],
                        cut_and_record, [SHIM], __file__, force)
    if manifest:  # compiled just now
        with open(os.path.join(OUT_DIR, "MANIFEST.txt"), "w") as fh:
            fh.write("reference functions compiled into libnerfshop_ref.so (file:first-last line, anchor)\n" + "\n".join(manifest) + "\n")
        if verbose:
            print("\n".join(manifest))
    return lib


def build_cuda(force: bool = False):
    """The same reference sources compiled by nvcc for sm_90a (oracle/ref_driver_cuda.cu): the reference's kernels and host loop
    run on the GPU. Returns the library path, or None when /root/reference is absent and no prebuilt library exists."""
    return build_library(LIB_CUDA, DRIVER_CUDA, "gen_cuda",
                         lambda gen: NVCC + ["-lineinfo", "-I", SHIM, "-I", gen, *REF_INCLUDES, DRIVER_CUDA, "-o", LIB_CUDA],
                         extract_all, [SHIM], __file__, force)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_cuda(force="--force" in sys.argv))
