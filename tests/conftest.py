import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
GOLDEN_CASES = ["id_deg3_64", "rigid_bg_96x64", "ragged_80x48_deg1", "precomp_init_70x50", "big_surfels_64",
                "near_cull_64", "single_32"]


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with `pytest -m gpu`)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if not has_gpu:
        skip = pytest.mark.skip(reason="no CUDA device")
        for it in items:
            if "gpu" in it.keywords:
                it.add_marker(skip)


@pytest.fixture(scope="session")
def built():
    """Make sure the CUDA library and the oracle are built (cheap if already up to date)."""
    from vidu4d_b200 import build as b
    b.build()
    from oracle import surfel_oracle
    surfel_oracle.build()
    return True


def load_golden(name):
    import numpy as np
    g = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    return {k: g[k] for k in g.files}


def oracle_forward_from_golden(g):
    from oracle import surfel_oracle as so
    P, W, H, deg, pre = [int(v) for v in g["in_meta"]]
    return so.forward(g["in_means3D"], g["in_opacities"], g["in_scales"], g["in_rotations"],
                      shs=None if pre else g["in_shs"], colors_precomp=g["in_colors_precomp"] if pre else None,
                      sh_degree=deg, W=W, H=H, tanfovx=float(g["in_tanfov"][0]), tanfovy=float(g["in_tanfov"][1]),
                      bg=g["in_bg"], viewmatrix=g["in_viewmatrix"], projmatrix=g["in_projmatrix"], campos=g["in_campos"])
