"""Import-name shim: GaussianEditor does ``from diff_gaussian_rasterization import GaussianRasterizationSettings,
GaussianRasterizer`` (gaussiansplatting/gaussian_renderer/__init__.py:14-17). With this repository on
``PYTHONPATH`` that import resolves to the H100-native implementation, so the reference's render()/GaussianModel
run unchanged."""
from gaussianeditor_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer,  # noqa: F401
                                            rasterize_gaussians, _RasterizeGaussians)
