"""gaussianeditor_b200 -- an H100-native (sm_90a) differentiable 3D-Gaussian-splatting rasterizer that drops in
behind GaussianEditor's ``gaussiansplatting/gaussian_renderer.render()``.

Only the one hot path is here (see DESIGN.md): ``csrc/`` holds the hand-written CUDA kernels behind a C ABI
(``include/gsr_b200.h``), ``rasterizer.py`` mirrors the reference's ``diff_gaussian_rasterization`` Python API,
``gaussian_renderer.py`` mirrors the render boundary, ``synth.py`` generates the seeded benchmark scenes.
"""
from .rasterizer import (GaussianRasterizationSettings, GaussianRasterizer,  # noqa: F401
                         rasterize_gaussians)
