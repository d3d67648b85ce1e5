"""similari_b200 -- H100-native association engine for Similari's cost-matrix + assignment hot path.

`similari_b200.engine`  array-level interface (numpy in / numpy out) over the C ABI of libsimilari_b200.so
`similari_b200.api`     the reference's Python class names (Sort, BatchSort, VisualSort, BatchVisualSort, nms, ...)
`similari_b200.workload` seeded synthetic workloads of the BASELINE configs
"""
from ._lib import (KIND_BATCH_SORT, KIND_BATCH_VISUAL_SORT, KIND_SORT, KIND_VISUAL_SORT, NONE_ID, POS_IOU, POS_MAHA,
                   VIS_COSINE, VIS_EUCLIDEAN, VOTING_POSITIONAL, VOTING_VISUAL, Options, Sb200Error, default_options)

__all__ = [
    "KIND_SORT", "KIND_BATCH_SORT", "KIND_VISUAL_SORT", "KIND_BATCH_VISUAL_SORT", "POS_MAHA", "POS_IOU", "VIS_EUCLIDEAN",
    "VIS_COSINE", "VOTING_VISUAL", "VOTING_POSITIONAL", "NONE_ID", "Options", "Sb200Error", "default_options",
]
