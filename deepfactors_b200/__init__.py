"""deepfactors_b200 -- H100-native (sm_90a) dense-alignment hot path of DeepFactors.

Only what the path needs: `csrc/` (CUDA kernels + the C ABI of include/dfk.h, built in-tree as
libdfk.so) and the host-side mirror of the reference's aligner interface (`aligners`).
`synth` and `se3` are numpy-only helpers (synthetic inputs, Sophus-convention pose algebra).
Heavy imports (torch) happen lazily on first use of `aligners`.
"""
from __future__ import annotations

import importlib

__all__ = ["aligners", "synth", "se3", "SfmAligner", "SE3Aligner"]
_LAZY = {"SfmAligner": "aligners", "SE3Aligner": "aligners", "DepthAligner": "aligners", "Window": "aligners", "SfmAlignerParams": "aligners",
         "DenseSfmParams": "aligners", "UpdateDepth": "aligners", "SobelGradients": "aligners",
         "GaussianBlurDown": "aligners", "SquaredError": "aligners", "ReprojectionLinearize": "aligners",
         "SparseGeometricLinearize": "aligners", "SparseGeometricLinearizeBatch": "aligners"}


def __getattr__(name):
    if name in ("aligners", "synth", "se3", "_lib"):
        return importlib.import_module("." + name, __name__)
    if name in _LAZY:
        return getattr(importlib.import_module("." + _LAZY[name], __name__), name)
    raise AttributeError(name)
