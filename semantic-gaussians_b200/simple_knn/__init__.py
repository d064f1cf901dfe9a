"""Drop-in for the reference's ``simple_knn`` extension (submodules/simple-knn): ``from simple_knn._C import
distCUDA2`` becomes ``from semantic_gaussians_b200.simple_knn._C import distCUDA2``."""
from ._C import distCUDA2  # noqa: F401
