"""AnnData-level drivers with the reference signatures (spateo/alignment/morpho_alignment.py:22-454).

The four public functions keep the reference's names, keyword arguments, defaults, return arity and the ``.obsm`` / ``.uns``
keys they write; the shared steps (input validation, key seeding, running one pair, storing its outputs) live in the small
helpers below.
"""

from __future__ import annotations

import os
import shutil
from pathlib import Path
from typing import List, Optional, Tuple, Union

import numpy as np

from ..anndata_lite import is_anndata_like
from .morpho_class import Morpho_pairwise
from .transform import BA_transform
from .utils import empty_cache, solve_RT_by_correspondence

Rep = Union[str, List[str]]


def _read_h5ad(path):
    try:
        import anndata as ad
    except ImportError as e:  # pragma: no cover - anndata is optional in this image
        raise ImportError("reading .h5ad files needs the `anndata` package") from e
    return ad.read_h5ad(path)


def _validate_models(models, models_path):
    """Input contract of the chain drivers (morpho_alignment.py:146-158, 249-261)."""
    if models_path is None:
        assert all(is_anndata_like(m) for m in models), "models should be a list of anndata if models_path is not given."
        return
    assert all(isinstance(m, str) for m in models), "models should be a list of file name if models_path is given."
    assert all(os.path.exists(os.path.join(models_path, m)) for m in models), "Some files in models_path do not exist."


def _working_copy(model):
    """The drivers never mutate their inputs (morpho_alignment.py:67): they work on copies. ``AnnDataLite`` copies share
    the (read-only) expression matrices; a real ``AnnData`` is copied with its own ``.copy()``."""
    from ..anndata_lite import AnnDataLite

    return model.copy(share_X=True) if isinstance(model, AnnDataLite) else model.copy()


def _seed_keys(slices, spatial_key, key_added):
    """Every slice starts with its raw coordinates under the three result keys (morpho_alignment.py:68-72)."""
    for sl in slices:
        for suffix in ("", "_rigid", "_nonrigid"):
            sl.obsm[key_added + suffix] = sl.obsm[spatial_key].copy()


def _solve_pair(fixed, moving, **solver_kwargs):
    """One ``Morpho_pairwise`` problem: ``moving`` is deformed onto ``fixed``. Returns (solver, P)."""
    solver = Morpho_pairwise(sampleA=moving, sampleB=fixed, **solver_kwargs)
    return solver, solver.run()


def _store_pair(target, solver, key_added, mode, iter_key_added, vecfld_key_added, coords=None):
    """Write one pair's outputs onto ``target`` (morpho_alignment.py:96-107). ``coords`` overrides the solver's own
    (rigid, non-rigid) coordinates (used when the field is carried over to a bigger slice)."""
    rigid, nonrigid = coords if coords is not None else (solver.optimal_RnA.copy(), solver.XAHat.copy())
    target.obsm[f"{key_added}_rigid"], target.obsm[f"{key_added}_nonrigid"] = rigid, nonrigid
    if mode == "SN-S":
        target.obsm[key_added] = target.obsm[f"{key_added}_rigid"]
    elif mode == "SN-N":
        target.obsm[key_added] = target.obsm[f"{key_added}_nonrigid"]
    if iter_key_added is not None:
        target.uns[iter_key_added] = solver.iter_added
    if vecfld_key_added is not None:
        target.uns[vecfld_key_added] = solver.vecfld


def _transfer_keys(kwargs) -> tuple:
    """The posterior-transfer keywords of a driver, (transfer_B, transfer_A): keys of the slices only, since an array would
    be ambiguous across the pairs of a chain."""
    keys = []
    for name in ("transfer_B", "transfer_A"):
        v = kwargs.get(name)
        if v is not None and not isinstance(v, str):
            raise ValueError(f"{name}: the drivers take the name of an .obsm matrix or .obs column of the slices; an array "
                             "is ambiguous across the pairs of a chain (pass arrays to Morpho_pairwise)")
        keys.append(v)
    return tuple(keys)


def _normalise_rows(x: np.ndarray, mass: np.ndarray) -> np.ndarray:
    """x / mass row by row (float64), rows of zero mass set to 0; float32 like the solver's outputs."""
    x, mass = np.asarray(x, dtype=np.float64), np.asarray(mass, dtype=np.float64).reshape(-1)
    out = np.zeros_like(x)
    ok = mass > 0
    out[ok] = x[ok] / mass[ok, None]
    return out.astype(np.float32)


def _store_transfer(fixed, moving, solver, key_B: Optional[str], key_A: Optional[str]):
    """Posterior-weighted features of one pair: ``moving.obsm[f"{key_B}_from_fixed"] = P_FB / K_NA`` and
    ``fixed.obsm[f"{key_A}_from_moving"] = PT_FA / K_NB``; for an ``.obs`` key also ``obs[...]`` = the category of the row
    maximum (missing for a row of zero mass)."""
    import pandas as pd

    for key, target, res, mass, cats, suffix in (
        (key_B, moving, solver.P_FB, solver.K_NA, solver.transfer_categories["B"], "_from_fixed"),
        (key_A, fixed, solver.PT_FA, solver.K_NB, solver.transfer_categories["A"], "_from_moving"),
    ):
        if key is None:
            continue
        norm = _normalise_rows(res, mass)
        target.obsm[key + suffix] = norm
        if cats is not None:
            codes = np.where(norm.max(axis=1) > 0, norm.argmax(axis=1), -1)
            target.obs[key + suffix] = pd.Categorical.from_codes(codes, categories=cats)


def morpho_align(
    models: List, rep_layer: Rep = "X", rep_field: Rep = "layer", genes: Optional[Union[List[str], np.ndarray]] = None,
    spatial_key: str = "spatial", key_added: str = "align_spatial", iter_key_added: Optional[str] = "iter_spatial",
    vecfld_key_added: str = "VecFld_morpho", mode: str = "SN-S", dissimilarity: Rep = "kl", max_iter: int = 200,
    dtype: str = "float32", device: str = "cpu", verbose: bool = True, **kwargs,
) -> Tuple[List, List[np.ndarray]]:
    """Serial alignment of consecutive slices; pair i+1 starts from pair i's aligned coordinates
    (morpho_alignment.py:22-111). Returns ``(align_models, pis)`` with ``pis[i] = P.T``.

    ``transfer_B`` / ``transfer_A`` (keys only): for every pair, the fixed slice's ``.obsm`` matrix / ``.obs`` column
    ``transfer_B`` carried to the moving slice through the pair's posterior, ``moving.obsm[f"{key}_from_fixed"] = P_FB /
    K_NA``, and the moving slice's ``transfer_A`` to the fixed one, ``fixed.obsm[f"{key}_from_moving"] = PT_FA / K_NB`` (rows
    of zero mass 0; an ``.obs`` key also gets ``obs[...]``, the category of the row maximum)."""
    transfer_keys = _transfer_keys(kwargs)
    aligned = [_working_copy(m) for m in models]
    _seed_keys(aligned, spatial_key, key_added)
    # the posterior of a pair whose cost matrix is streamed (too large for the device) is not built: its entry of pis is None
    kwargs.setdefault("materialize_P", "auto")
    pis = []
    for fixed, moving in zip(aligned[:-1], aligned[1:]):
        solver, P = _solve_pair(
            fixed, moving, rep_layer=rep_layer, rep_field=rep_field, dissimilarity=dissimilarity, genes=genes,
            spatial_key=key_added, key_added=key_added, iter_key_added=iter_key_added, vecfld_key_added=vecfld_key_added,
            max_iter=max_iter, dtype=dtype, device=device, verbose=verbose, **kwargs,
        )
        _store_pair(moving, solver, key_added, mode, iter_key_added, vecfld_key_added)
        _store_transfer(fixed, moving, solver, *transfer_keys)
        pis.append(None if P is None else P.T)
        del solver
        empty_cache(device=device)
    return aligned, pis


def pair_transformation(modelA, modelB, spatial_key="spatial", **pairwise_kwargs) -> dict:
    """One link of the chain: align ``modelB`` (moving) onto ``modelA`` (fixed) on RAW coordinates and return the 2-D
    similarity that maps B's raw coordinates onto the aligned ones (morpho_alignment.py:189-211)."""
    pairwise_kwargs.setdefault("materialize_P", False)
    solver, _ = _solve_pair(modelA, modelB, spatial_key=spatial_key, **pairwise_kwargs)
    R, t = solve_RT_by_correspondence(solver.optimal_RnA[:, :2], np.asarray(modelB.obsm[spatial_key])[:, :2])
    return {"Rotation": R, "Translation": t}


def morpho_align_transformation(
    models: List, models_path: Optional[str] = None, save_transformation: bool = False,
    transformation_path: Optional[str] = "./Spateo_transformation", resume: bool = False, rep_layer: Rep = "X",
    rep_field: Rep = "layer", genes: Optional[Union[List[str], np.ndarray]] = None, spatial_key: str = "spatial",
    key_added: str = "align_spatial", iter_key_added: Optional[str] = "iter_spatial",
    vecfld_key_added: str = "VecFld_morpho", dissimilarity: Rep = "kl", max_iter: int = 200, dtype: str = "float32",
    device: str = "cpu", verbose: bool = True, **kwargs,
):
    """Independent pairwise alignments on raw coordinates -> list of {"Rotation", "Translation"} with optional
    per-pair ``.npy`` checkpoints and resume (morpho_alignment.py:114-218)."""
    _validate_models(models, models_path)
    from_disk = models_path is not None
    n_pairs = len(models) - 1
    checkpoint = (lambda i: os.path.join(transformation_path, f"transformation_{i}.npy"))
    first, done = 0, []
    if save_transformation:
        Path(transformation_path).mkdir(parents=True, exist_ok=True)
        if not resume:
            remove_all_files_in_directory(transformation_path)
        else:
            # Restart at the highest pair index that has a checkpoint and recompute that pair, as the reference does
            # (morpho_alignment.py:166-179) — but keep only the links BEFORE it, as plain dicts: the reference appends
            # the re-computed pair on top of its own loaded copy (and its np.load lacks allow_pickle), which leaves
            # len(models) entries and breaks morpho_align_apply_transformation.
            have = [i for i in range(n_pairs) if os.path.exists(checkpoint(i))]
            first = max(have) if have else 0
            missing = [i for i in range(first) if i not in have]
            if missing:
                raise FileNotFoundError(f"resume: checkpoints of pairs {missing} are missing in {transformation_path}")
            done = [_as_link(np.load(checkpoint(i), allow_pickle=True)) for i in range(first)]
    load = (lambda k: _read_h5ad(os.path.join(models_path, models[k]))) if from_disk else (lambda k: models[k])
    fixed = load(first)
    for i in range(first, n_pairs):
        moving = load(i + 1)
        link = pair_transformation(
            fixed, moving, spatial_key=spatial_key, rep_layer=rep_layer, rep_field=rep_field, dissimilarity=dissimilarity,
            genes=genes, key_added=key_added, iter_key_added=iter_key_added, vecfld_key_added=vecfld_key_added,
            max_iter=max_iter, dtype=dtype, device=device, verbose=verbose, **kwargs,
        )
        done.append(link)
        if save_transformation:
            np.save(checkpoint(i), link)
        fixed = moving
    return done


def _as_link(tr) -> dict:
    """A checkpoint loaded with ``np.load(..., allow_pickle=True)`` is a 0-d object array around the dict."""
    return tr.item() if isinstance(tr, np.ndarray) and tr.dtype == object else tr


def compose_transformations(transformation: List[dict]):
    """Serial prefix composition of per-pair similarities (morpho_alignment.py:274-301):
    ``cur_t = t_i @ cur_R.T + cur_t ; cur_R = cur_R @ R_i``. Returns the cumulative (R, t) of slices 1..n-1."""
    cur_R, cur_t = np.diag((1.0, 1.0)), np.zeros((2,))
    out = []
    for tr in transformation:
        tr = _as_link(tr)
        cur_t = tr["Translation"] @ cur_R.T + cur_t
        cur_R = cur_R @ tr["Rotation"]
        out.append((cur_R.copy(), cur_t.copy()))
    return out


def morpho_align_apply_transformation(
    models: List, models_path: Optional[str] = None, transformation: List[dict] = None,
    transformation_path: Optional[str] = "./Spateo_transformation", spatial_key: str = "spatial",
    key_added: str = "align_spatial", save_models_path: Optional[str] = None, verbose: bool = True,
):
    """Apply the composed chain of 2-D similarities to every slice (morpho_alignment.py:221-314)."""
    _validate_models(models, models_path)
    from_disk = models_path is not None
    if transformation is not None:
        assert len(transformation) == len(models) - 1, "The length of transformation should be len(models) - 1."
    else:
        assert os.path.exists(transformation_path), "transformation_path does not exist."
        transformation = [
            np.load(os.path.join(transformation_path, f"transformation_{i}.npy"), allow_pickle=True)
            for i in range(len(models) - 1)
        ]
    if save_models_path is not None:
        Path(save_models_path).mkdir(parents=True, exist_ok=True)
    # slice 0 keeps its coordinates; slice k gets the composition of links 0..k-1
    placements = [(np.diag((1.0, 1.0)), np.zeros((2,)))] + compose_transformations(transformation)
    kept = []
    for k, (R_k, t_k) in enumerate(placements):
        sl = _read_h5ad(os.path.join(models_path, models[k])) if from_disk else models[k]
        raw = sl.obsm[spatial_key].copy()
        sl.obsm[key_added] = raw if k == 0 else raw @ R_k.T + t_k
        if save_models_path is not None:
            sl.write(os.path.join(save_models_path, models[k]))
        elif from_disk:
            kept.append(sl)
    return kept if from_disk else models


def morpho_align_ref(
    models: List, models_ref: Optional[List] = None, n_sampling: Optional[int] = 2000, sampling_method: str = "random",
    rep_layer: Rep = "X", rep_field: Rep = "layer", genes: Optional[Union[list, np.ndarray]] = None,
    spatial_key: str = "spatial", key_added: str = "align_spatial", iter_key_added: Optional[str] = "iter_spatial",
    vecfld_key_added: Optional[str] = "VecFld_morpho", mode: str = "SN-S", dissimilarity: Rep = "kl",
    max_iter: int = 200, dtype: str = "float32", device: str = "cpu", verbose: bool = True, **kwargs,
):
    """Align down-sampled reference models, then carry the learned field to the full models with ``BA_transform``
    (morpho_alignment.py:318-454). Down-sampling: the reference delegates to third-party ``dynamo.tools.sampling``
    (absent); only ``sampling_method="random"`` is provided here."""
    if models_ref is None:
        if sampling_method != "random":
            raise NotImplementedError("only sampling_method='random' is available (dynamo's trn/kmeans samplers are third-party)")
        models_ref = []
        for m in models:
            n = m.shape[0]
            models_ref.append(m[np.sort(np.random.choice(n, min(n_sampling, n), replace=False))].copy())
    full = [_working_copy(m) for m in models]
    small = [_working_copy(m) for m in models_ref]
    _seed_keys(full + small, spatial_key, key_added)
    pis, pis_ref = [], []
    for i in range(len(full) - 1):
        solver, P = _solve_pair(
            small[i], small[i + 1], rep_layer=rep_layer, rep_field=rep_field, dissimilarity=dissimilarity, genes=genes,
            spatial_key=key_added, key_added=key_added, iter_key_added=iter_key_added, vecfld_key_added=vecfld_key_added,
            max_iter=max_iter, dtype=dtype, device=device, verbose=verbose, **kwargs,
        )
        _store_pair(small[i + 1], solver, key_added, mode, iter_key_added, vecfld_key_added)
        # the same field evaluated on every cell of the full slice
        nonrigid, _, rigid = BA_transform(vecfld=solver.vecfld, quary_points=full[i + 1].obsm[key_added], device=device,
                                          dtype=dtype)
        _store_pair(full[i + 1], solver, key_added, mode, iter_key_added, vecfld_key_added, coords=(rigid, nonrigid))
        pis_ref.append(P)
        pis.append(P)
    return full, small, pis, pis_ref


def remove_all_files_in_directory(directory_path):
    if not os.path.exists(directory_path):
        return
    for name in os.listdir(directory_path):
        fp = os.path.join(directory_path, name)
        if os.path.isdir(fp) and not os.path.islink(fp):
            shutil.rmtree(fp)
        else:
            os.unlink(fp)
