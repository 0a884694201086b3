"""spateo_release_b200 — H100-native (sm_90a) implementation of Spateo's pairwise morpho-alignment hot path.

``import spateo_release_b200 as st`` exposes the reference's namespaces for this path: ``st.align.morpho_align`` /
``Morpho_pairwise`` / ``BA_transform`` and ``st.tdr.morphofield_gp`` / ``morphofield_sparsevfc`` / ``morphofield``.
The array math runs in ``libspateo_b200.so`` (hand-written CUDA, C ABI in ``include/spateo_b200.h``); there is no CPU
fallback.
"""

from . import alignment as align
from . import tdr
from .anndata_lite import AnnDataLite

__all__ = ["align", "tdr", "AnnDataLite"]
