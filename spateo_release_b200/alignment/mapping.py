"""Optimal cell-to-cell mapping from an alignment posterior (reference: spateo/alignment/utils.py:157-254).

The reference scans a dense ``pi`` on the host (``np.argwhere(pi == pi.max(axis))``). Here the row / column maxima come
from the device: either from the fused ``spb_posterior_argmax_mapped`` kernels, which read the resident cost matrix once and
never form P (``Morpho_pairwise(..., compute_mapping=True).mapping`` -> :class:`ArgmaxPi`), or — for a dense ``pi`` the
caller already holds — from chunked torch reductions on the GPU. Ties (several entries equal to the maximum; with
floating-point posteriors that means an all-zero row or column) are broken with a KD-tree on the coordinates exactly as
the reference does.
"""

from __future__ import annotations

from typing import Tuple

import numpy as np
import pandas as pd
from scipy.spatial import cKDTree

from .. import _capi


class ArgmaxPi:
    """Row and column maxima of a posterior that was never materialised (shape ``(n_rows, n_cols)``).

    ``row_arg[i]`` / ``row_val[i]``: lowest column index and value of the maximum of row i; ``col_arg`` / ``col_val``
    likewise per column. ``.T`` swaps the roles (the drivers hand ``P.T`` to the mapping helpers).

    Tie-breaking differs from the reference for equal NON-ZERO maxima (exact duplicates: cells with identical coordinates
    and expression): ``get_optimal_mapping_relationship`` (spateo/alignment/utils.py:157-191) resolves such ties with a
    KD-tree over the coordinates. Here a row's tie goes to the lowest column index, and a column's tie to the moving cell that
    comes first in the solver's processing order (the k-d order of ``kd_order``), not the lowest input index. Ties at value 0
    (rows / columns without any posterior mass) are handled like the reference. Pass a dense ``pi`` to get the reference's
    tie rule."""

    def __init__(self, shape, row_arg, row_val, col_arg, col_val):
        self.shape = tuple(shape)
        self.row_arg, self.row_val = np.asarray(row_arg, dtype=np.int64), np.asarray(row_val)
        self.col_arg, self.col_val = np.asarray(col_arg, dtype=np.int64), np.asarray(col_val)

    @property
    def T(self) -> "ArgmaxPi":
        return ArgmaxPi((self.shape[1], self.shape[0]), self.col_arg, self.col_val, self.row_arg, self.row_val)

    def copy(self) -> "ArgmaxPi":
        return ArgmaxPi(self.shape, self.row_arg.copy(), self.row_val.copy(), self.col_arg.copy(), self.col_val.copy())

    @staticmethod
    def decode(keys: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        """(argmax, value) from the packed ``spb_posterior_argmax_mapped`` keys."""
        keys = np.asarray(keys, dtype=np.uint64)
        val = (keys >> np.uint64(32)).astype(np.uint32).view(np.float32)
        arg = (np.uint64(0xFFFFFFFF) - (keys & np.uint64(0xFFFFFFFF))).astype(np.int64)
        return arg, val


def _dense_maxima(pi: np.ndarray, chunk_bytes: int = 1 << 30):
    """Row/column maxima, first arg-maxima and tie counts of a dense host matrix, reduced on the GPU in row chunks."""
    import torch

    _capi.require_cuda()
    n, m = pi.shape
    dev = torch.device("cuda")
    rows_per = max(1, int(chunk_bytes // max(1, m * pi.dtype.itemsize)))
    row_val = np.empty(n, dtype=pi.dtype)
    row_arg = np.empty(n, dtype=np.int64)
    row_cnt = np.empty(n, dtype=np.int64)
    col_val = torch.full((m,), -float("inf"), dtype=torch.from_numpy(pi[:1]).dtype, device=dev)
    col_arg = torch.zeros((m,), dtype=torch.int64, device=dev)
    chunks = []
    keep = pi.nbytes <= (8 << 30)  # keep the uploaded chunks for the tie-count pass when they fit comfortably
    for i0 in range(0, n, rows_per):
        t = torch.from_numpy(np.ascontiguousarray(pi[i0 : i0 + rows_per])).to(dev)
        v, a = t.max(dim=1)
        row_val[i0 : i0 + len(v)] = v.cpu().numpy()
        row_cnt[i0 : i0 + len(v)] = (t == v[:, None]).sum(1).cpu().numpy()
        # lowest index among equal maxima, like np.argwhere order
        first = torch.where(t == v[:, None], torch.arange(m, device=dev)[None, :], m).min(dim=1).values
        row_arg[i0 : i0 + len(v)] = first.cpu().numpy()
        cv, ca = t.max(dim=0)
        cfirst = torch.where(t == cv[None, :], torch.arange(len(t), device=dev)[:, None], len(t)).min(dim=0).values
        better = cv > col_val
        col_arg = torch.where(better, cfirst + i0, col_arg)
        col_val = torch.where(better, cv, col_val)
        if keep:
            chunks.append((i0, t))
    col_cnt = torch.zeros((m,), dtype=torch.int64, device=dev)
    if keep:
        for i0, t in chunks:
            col_cnt += (t == col_val[None, :]).sum(0)
    else:
        for i0 in range(0, n, rows_per):
            t = torch.from_numpy(np.ascontiguousarray(pi[i0 : i0 + rows_per])).to(dev)
            col_cnt += (t == col_val[None, :]).sum(0)
    return (row_val, row_arg, row_cnt, col_val.cpu().numpy(), col_arg.cpu().numpy(), col_cnt.cpu().numpy())


def _assemble(arg, cnt, candidates_of, own_pts, other_pts, keep_all, key_first: bool):
    """Index pairs of one axis: single maxima first (ascending), then the tied keys resolved by the nearest coordinate
    (utils.py:166-185); ``keep_all`` lists every tied candidate in argwhere order instead."""
    n = len(arg)
    idx = np.arange(n)
    single = cnt == 1
    pair = (lambda k, o: (k, o)) if key_first else (lambda k, o: (o, k))
    if keep_all:
        parts = [np.stack(pair(idx[single], arg[single]), axis=1)]
        for i in idx[~single]:
            c = candidates_of(i)
            parts.append(np.stack(pair(np.full(len(c), i), c), axis=1))
        out = np.concatenate(parts, axis=0)
        order = np.lexsort((out[:, 1], out[:, 0]))
        return out[order]
    out = np.stack(pair(idx[single], arg[single]), axis=1)
    out = out[np.lexsort((out[:, 1], out[:, 0]))]  # np.argwhere order of the reference (row-major)
    extra = []
    for i in idx[~single]:
        c = candidates_of(i)
        _, ii = cKDTree(other_pts[c]).query(own_pts[i], k=1)
        extra.append(pair(i, c[ii]))
    if extra:
        out = np.concatenate([out, np.asarray(extra, dtype=out.dtype).reshape(-1, 2)], axis=0)
    return out


def get_optimal_mapping_relationship(X: np.ndarray, Y: np.ndarray, pi, keep_all: bool = False):
    """utils.py:157-191. ``pi``: dense ``[len(X), len(Y)]`` array, or an :class:`ArgmaxPi`.

    Returns ``X_max_index [n, 2]``, ``X_pi_value [n, 1]``, ``Y_max_index``, ``Y_pi_value`` like the reference."""
    X, Y = np.asarray(X), np.asarray(Y)
    if isinstance(pi, ArgmaxPi):
        n, m = pi.shape
        # exact ties between floating-point posteriors only occur at 0 (an empty row / column): every entry ties
        row_cnt = np.where(pi.row_val > 0, 1, m)
        col_cnt = np.where(pi.col_val > 0, 1, n)
        row_c = lambda i: np.arange(m)
        col_c = lambda j: np.arange(n)
        row_val, row_arg, col_val, col_arg = pi.row_val, pi.row_arg, pi.col_val, pi.col_arg
        value = None
    else:
        if hasattr(pi, "toarray"):
            raise TypeError("get_optimal_mapping_relationship needs a dense pi or an ArgmaxPi; call .toarray() first.")
        pi = np.asarray(pi)
        row_val, row_arg, row_cnt, col_val, col_arg, col_cnt = _dense_maxima(pi)
        row_c = lambda i: np.flatnonzero(pi[i] == row_val[i])
        col_c = lambda j: np.flatnonzero(pi[:, j] == col_val[j])
        value = pi
    X_max_index = _assemble(row_arg, row_cnt, row_c, X, Y, keep_all, key_first=True)
    Y_max_index = _assemble(col_arg, col_cnt, col_c, Y, X, keep_all, key_first=False)
    if value is not None:
        X_pi_value = value[X_max_index[:, 0], X_max_index[:, 1]].reshape(-1, 1)
        Y_pi_value = value[Y_max_index[:, 0], Y_max_index[:, 1]].reshape(-1, 1)
    else:
        X_pi_value = row_val[X_max_index[:, 0]].reshape(-1, 1)
        Y_pi_value = col_val[Y_max_index[:, 1]].reshape(-1, 1)
    return X_max_index, X_pi_value, Y_max_index, Y_pi_value


def mapping_aligned_coords(X: np.ndarray, Y: np.ndarray, pi, keep_all: bool = False) -> Tuple[dict, dict]:
    """utils.py:194-254 — two dicts (anchored on X and on Y) with ``mapping_X``, ``mapping_Y``, ``pi_index``, ``pi_value``."""
    X, Y = np.asarray(X).copy(), np.asarray(Y).copy()
    X_max_index, X_pi_value, Y_max_index, Y_pi_value = get_optimal_mapping_relationship(X=X, Y=Y, pi=pi, keep_all=keep_all)
    mappings = []
    for max_index, pi_value, subset in ((X_max_index, X_pi_value, "index_x"), (Y_max_index, Y_pi_value, "index_y")):
        data = pd.DataFrame(np.concatenate([max_index, pi_value], axis=1), columns=["index_x", "index_y", "pi_value"])
        data = data.astype({"index_x": np.int32, "index_y": np.int32, "pi_value": np.float64})
        data.sort_values(by=[subset, "pi_value"], ascending=[True, False], inplace=True)
        data.drop_duplicates(subset=[subset], keep="first", inplace=True)
        mappings.append(
            {
                "mapping_X": X[data["index_x"].values],
                "mapping_Y": Y[data["index_y"].values],
                "pi_index": data[["index_x", "index_y"]].values,
                "pi_value": data["pi_value"].values,
            }
        )
    return mappings[0], mappings[1]
