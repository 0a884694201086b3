"""TEST INFRASTRUCTURE ONLY — imports the UNMODIFIED reference (SURVEY.md Appendix C) from the spateo-release checkout
named by the environment variable ``SPATEO_REFERENCE``.

Only usable where such a checkout exists; the test suite does not need it. It is used by
``tests/golden/make_golden.py`` to generate the committed golden fixtures and by ``oracle/check_oracle_vs_reference.py``
to pin the numpy restatement in ``oracle/morpho_oracle.py`` against the real thing. Nothing in the product package,
``bench.py`` or the ``-m gpu`` tests imports this module.

Mechanics: ``anndata`` is not installed, so a stub module exposing ``AnnData = AnnDataLite`` is registered; the
package ``__init__`` files of ``spateo.alignment`` / ``spateo.alignment.methods`` import pyvista/POT (absent), so bare
package modules are pre-registered and only ``methods/{backend,utils,morpho_class}.py`` are imported (unmodified).
"""

import importlib
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("SPATEO_REFERENCE", "")


def reference_available() -> bool:
    return bool(REFERENCE_ROOT) and os.path.isdir(os.path.join(REFERENCE_ROOT, "spateo", "alignment", "methods"))


_loaded = {}


def load_reference():
    """Return (morpho_class_module, utils_module) of the unmodified reference."""
    if "mc" in _loaded:
        return _loaded["mc"], _loaded["utils"]
    if not reference_available():
        raise RuntimeError("reference tree not present: set SPATEO_REFERENCE to a spateo-release checkout")
    repo_root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if repo_root not in sys.path:
        sys.path.insert(0, repo_root)
    from spateo_release_b200.anndata_lite import AnnDataLite

    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)

    if "anndata" not in sys.modules:

        class _Stub(types.ModuleType):
            def __getattr__(self, n):
                if n.startswith("__"):
                    raise AttributeError(n)
                return lambda *a, **k: None

        ad = _Stub("anndata")
        ad.AnnData = AnnDataLite
        sys.modules["anndata"] = ad

    import spateo  # noqa: F401  (lazy loaders only)

    for name, path in [
        ("spateo.alignment", os.path.join(REFERENCE_ROOT, "spateo/alignment")),
        ("spateo.alignment.methods", os.path.join(REFERENCE_ROOT, "spateo/alignment/methods")),
    ]:
        if name not in sys.modules:
            pkg = types.ModuleType(name)
            pkg.__path__ = [path]
            sys.modules[name] = pkg
    mc = importlib.import_module("spateo.alignment.methods.morpho_class")
    utils = importlib.import_module("spateo.alignment.methods.utils")
    _loaded["mc"], _loaded["utils"] = mc, utils
    return mc, utils


def load_reference_tdr():
    """Return (gaussian_process_module, GPVectorField_module) of the unmodified reference's st.tdr morphofield code.

    ``spateo.tdr``'s package ``__init__`` pulls pyvista & co, so bare packages are registered and only the two leaf
    modules are imported; ``numpy.matlib`` is imported first because the reference's ``_con_K(return_d=True)`` uses
    ``np.matlib.tile`` without importing it (gaussian_process.py:28)."""
    if "gp" in _loaded:
        return _loaded["gp"], _loaded["gpvf"]
    load_reference()
    import numpy.matlib  # noqa: F401

    for name, rel in [
        ("spateo.tdr", "spateo/tdr"),
        ("spateo.tdr.morphometrics", "spateo/tdr/morphometrics"),
        ("spateo.tdr.morphometrics.morphofield", "spateo/tdr/morphometrics/morphofield"),
        ("spateo.tdr.morphometrics.morphofield_dg", "spateo/tdr/morphometrics/morphofield_dg"),
    ]:
        if name not in sys.modules:
            pkg = types.ModuleType(name)
            pkg.__path__ = [os.path.join(REFERENCE_ROOT, rel)]
            sys.modules[name] = pkg
    if "spateo.tdr.interpolations" not in sys.modules:
        interp = types.ModuleType("spateo.tdr.interpolations")
        interp.get_X_Y_grid = lambda *a, **k: None
        sys.modules["spateo.tdr.interpolations"] = interp
    gp = importlib.import_module("spateo.tdr.morphometrics.morphofield.gaussian_process")
    gpvf = importlib.import_module("spateo.tdr.morphometrics.morphofield_dg.GPVectorField")
    _loaded["gp"], _loaded["gpvf"] = gp, gpvf
    return gp, gpvf


def load_reference_align_utils():
    """The unmodified ``spateo/alignment/utils.py`` (get_optimal_mapping_relationship, mapping_aligned_coords)."""
    if "au" in _loaded:
        return _loaded["au"]
    load_reference()
    _loaded["au"] = importlib.import_module("spateo.alignment.utils")
    return _loaded["au"]


def load_reference_transform():
    """The unmodified ``spateo/alignment/transform.py`` (BA_transform). Its ``from .methods import ...`` list is served from
    the already-imported ``methods.utils`` module; names that no longer exist upstream are bound to ``None``."""
    if "tr" in _loaded:
        return _loaded["tr"]
    _, utils = load_reference()
    pkg = sys.modules["spateo.alignment.methods"]
    for name in ("_chunk", "_data", "_dot", "_mul", "_pi", "_power", "_prod", "_unsqueeze", "cal_dist", "cal_dot",
                 "calc_exp_dissimilarity", "check_backend", "check_exp", "con_K", "filter_common_genes", "intersect_lsts"):
        if not hasattr(pkg, name):
            setattr(pkg, name, getattr(utils, name, None))
    _loaded["tr"] = importlib.import_module("spateo.alignment.transform")
    return _loaded["tr"]


def load_reference_drivers():
    """The unmodified ``spateo/alignment/morpho_alignment.py`` (morpho_align, morpho_align_transformation,
    morpho_align_apply_transformation). Its ``from spateo.alignment.methods import Morpho_pairwise, empty_cache`` is served
    from the already-imported leaf modules; ``spateo.alignment.transform`` / ``utils`` are imported unmodified."""
    if "drv" in _loaded:
        return _loaded["drv"]
    mc, utils = load_reference()
    load_reference_transform()
    pkg = sys.modules["spateo.alignment.methods"]
    pkg.Morpho_pairwise = mc.Morpho_pairwise
    pkg.empty_cache = utils.empty_cache
    _loaded["drv"] = importlib.import_module("spateo.alignment.morpho_alignment")
    return _loaded["drv"]
