"""Drop-in `r3dg_rasterization` package: put `<repo>/dropin` (and `<repo>`) on PYTHONPATH and the
reference's own wrapper — gaussian_renderer/r3dg_rasterization.py:8 `from r3dg_rasterization import _C`
— picks up this project's kernels instead of JIT-compiling the reference sources.  The class / function
names of the reference's packaged wrapper (r3dg-rasterization/r3dg_rasterization/__init__.py) are
re-exported too, so `from r3dg_rasterization import GaussianRasterizer` keeps working."""
from relightable3dgaussian_b200 import _C_raster as _C  # noqa: F401
from relightable3dgaussian_b200.rasterizer import (  # noqa: F401
    GaussianRasterizationSettings, GaussianRasterizer, rasterize_gaussians)
