import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: `pytest -m gpu`)")


@pytest.fixture(scope="session")
def scene():
    """Seeded synthetic fox-scale scene: model params, occupancy bitfield (nerfshop_b200/synthetic.py)."""
    from nerfshop_b200 import synthetic as syn

    model = syn.make_model(seed=1337)
    occ = syn.make_occupancy(model)
    return model, occ


@pytest.fixture(scope="session")
def oracle(scene):
    from oracle import oracle as orc

    model, occ = scene
    return orc.Oracle(model.desc, model.params, occ)


@pytest.fixture(scope="session")
def built_lib():
    """The sm_90a library, built in-tree if needed (nvcc cross-compiles without a GPU)."""
    from nerfshop_b200 import build

    return build.build()


@pytest.fixture(scope="session")
def renderer(scene, built_lib):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nerfshop_b200.renderer import NerfRenderer

    model, occ = scene
    r = NerfRenderer(0)
    r.upload_model(model.desc, model.params)
    r.upload_occupancy(occ)
    yield r
    r.close()


def random_coords(n, seed=0):
    """n NerfCoordinate rows {pos3 in [0,1], dt, dir3 in [0,1]} (nerf.h:73)."""
    rng = np.random.default_rng(seed)
    c = np.zeros((n, 7), np.float32)
    c[:, :3] = rng.random((n, 3), dtype=np.float32)
    c[:, 3] = rng.random(n, dtype=np.float32)
    d = rng.standard_normal((n, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    c[:, 4:] = (d + 1.0) * 0.5
    return c
