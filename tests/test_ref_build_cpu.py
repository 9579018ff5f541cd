"""The rebuild rule of the reference libraries under oracle/_ref (oracle/ref_build.py): each library is rebuilt when one of the repository's
files it is built from is newer than it. Every library's build() is run with ref_build.build_library replaced by a recorder, so the files
checked are those the library's own declaration derives; nothing is compiled, and the reference's sources need not exist."""
import os

import pytest

from oracle import ref_build, ref_camera_build, ref_mesh_build, ref_mesh_opt_build, ref_slices_build, ref_vanish_build, ref_video_build

ORACLE = os.path.dirname(os.path.abspath(ref_build.__file__))
RENDER_PATH = [os.path.join(ORACLE, "ref_common.inl"), os.path.join(os.path.dirname(ORACLE), "include", "nerfshop_b200.h")]

# library: (build module, build function, stand-in directories, further files it includes)
LIBRARIES = {
    "libnerfshop_ref.so": (ref_build, ref_build.build, ["ref_shim"], RENDER_PATH),
    "libnerfshop_ref_cuda.so": (ref_build, ref_build.build_cuda, ["ref_shim"], RENDER_PATH),
    "libnerfshop_ref_mesh_cuda.so": (ref_mesh_build, ref_mesh_build.build, ["ref_shim_mesh", "ref_shim"], []),
    "libnerfshop_ref_mesh_opt_cuda.so": (ref_mesh_opt_build, ref_mesh_opt_build.build, ["ref_shim"], []),
    "libnerfshop_ref_slices_cuda.so": (ref_slices_build, ref_slices_build.build, ["ref_shim_slices", "ref_shim"], []),
    "libnerfshop_ref_video_cuda.so": (ref_video_build, ref_video_build.build, ["ref_shim"], RENDER_PATH + [ref_build.DRIVER_CUDA]),
    "libnerfshop_ref_vanish.so": (ref_vanish_build, ref_vanish_build.build, ["ref_shim"], RENDER_PATH + [ref_build.DRIVER]),
    "libnerfshop_ref_camera.so": (ref_camera_build, ref_camera_build.build, ["ref_shim_camera"], []),
}


def _files_under(d):
    return [os.path.join(root, f) for root, _, files in os.walk(os.path.join(ORACLE, d)) for f in files]


@pytest.mark.parametrize("name", list(LIBRARIES))
def test_dependencies_of_every_library(monkeypatch, name):
    module, build, shim_dirs, includes = LIBRARIES[name]
    calls = []
    monkeypatch.setattr(ref_build, "build_library", lambda lib, driver, gen_name, compile_cmd, cut, shims, mod, force=False:
                        calls.append((lib, driver, shims, mod)))
    build()
    assert len(calls) == 1
    lib, driver, shims, mod = calls[0]
    assert os.path.basename(lib) == name
    deps = ref_build.dependencies(driver, shims, mod)
    shim_files = [f for d in shim_dirs for f in _files_under(d)]
    assert shim_files
    expected = [driver, os.path.abspath(ref_build.__file__), os.path.abspath(module.__file__)] + shim_files + includes
    missing = [f for f in expected if os.path.normpath(f) not in deps]
    assert not missing, missing


def test_stale_when_any_dependency_is_newer(tmp_path):
    lib = tmp_path / "lib.so"
    deps = [tmp_path / "driver.cu", tmp_path / "shim.h"]
    for p in deps:
        p.write_text("")
        os.utime(p, (1000, 1000))
    assert ref_build.stale(str(lib), deps)
    lib.write_text("")
    os.utime(lib, (1000, 1000))
    assert not ref_build.stale(str(lib), deps)
    os.utime(lib, (2000, 2000))
    assert not ref_build.stale(str(lib), deps)
    for p in deps:
        os.utime(p, (2001, 2001))
        assert ref_build.stale(str(lib), deps)
        os.utime(p, (1000, 1000))
