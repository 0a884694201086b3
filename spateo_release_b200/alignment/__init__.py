"""``st.align`` namespace of the H100-native hot path (reference: spateo/alignment/__init__.py:1-29)."""

from .morpho_alignment import (
    compose_transformations,
    morpho_align,
    morpho_align_apply_transformation,
    morpho_align_ref,
    morpho_align_transformation,
    pair_transformation,
)
from .morpho_class import Morpho_pairwise
from .transform import BA_transform, field_eval
from .utils import empty_cache, solve_RT_by_correspondence
from .distributed import (align_chain_pipelined, column_block, gather_transformations, morpho_align_chain_sharded,
                          morpho_align_column_sharded, morpho_align_pair_sharded, shard_pairs)
from .mapping import ArgmaxPi, get_optimal_mapping_relationship, mapping_aligned_coords
