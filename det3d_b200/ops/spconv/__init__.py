"""H100-native stand-in for the `spconv` (v1.x) package surface Det3D uses."""
from .core import (ConvWeights, Rulebook, SparseLevel, build_conv_rulebook, build_subm_rulebook,
                   alloc_conv_rulebook, alloc_subm_rulebook, level_from_coors, sparse_conv,
                   sparse_to_dense)
from .fused import FusedSparseEncoder, compile_plan
from .modules import (SparseConv3d, SparseConvolution, SparseConvTensor, SparseModule,
                      SparseSequential, SubMConv3d)

__all__ = [
    "SparseConvTensor", "SparseModule", "SparseSequential", "SparseConvolution", "SparseConv3d",
    "SubMConv3d", "FusedSparseEncoder", "compile_plan", "ConvWeights", "Rulebook", "SparseLevel",
    "build_conv_rulebook", "build_subm_rulebook", "alloc_conv_rulebook", "alloc_subm_rulebook",
    "level_from_coors", "sparse_conv", "sparse_to_dense",
]
