"""Drop-in shim: `from diff_surfel_rasterization import GaussianRasterizationSettings, GaussianRasterizer`
(gs/gaussian_renderer/__init__.py:14 of yikaiw/Vidu4D) resolves to the H100-native implementation when this
repository's root is on sys.path ahead of the reference package."""
from vidu4d_b200.rasterizer import (  # noqa: F401
    GaussianRasterizationSettings,
    GaussianRasterizer,
    _RasterizeGaussians,
    cpu_deep_copy_tuple,
    rasterize_gaussians,
)
from . import _C  # noqa: F401  (importable submodule, like the reference's pybind extension)
