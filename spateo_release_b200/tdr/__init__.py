"""``st.tdr`` entry points that share the Gaussian-kernel vector field (reference: spateo/tdr/__init__.py)."""

from .interpolations import kernel_interpolation
from .morphofield import morphofield, morphofield_gp, morphofield_sparsevfc
from .morphofield_dg import (
    GPVectorField,
    Jacobian_GP_gaussian_kernel,
    morphofield_acceleration,
    morphofield_curl,
    morphofield_curvature,
    morphofield_divergence,
    morphofield_jacobian,
    morphofield_torsion,
    morphofield_velocity,
)
from .morphopath import morphopath
