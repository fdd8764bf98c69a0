"""dim-b200: the H100-native (sm_90a) hot path of 3DOM-FBK/deep-image-matching behind the reference's plugin API.

The directory name ``deep-image-matching_b200`` is fixed by the project layout and is not a Python identifier;
``dim_b200`` (repo root) is a two-line package whose ``__path__`` points here, so ``import dim_b200.extractors.superpoint``
imports this package's modules under that name.
"""
__version__ = "0.2.0"
