"""GPU: the K^T P K contraction kernels (morpho_class.py:1266-1279; SparseVFC normal equations) against float64 numpy.

``spb_gram_tc`` = wgmma / TMA kernel with the 3xTF32 split on the row-centred kernel (fp32-accurate products, fp32
accumulation over at most 4096 reduction elements, fp64 fold and rank-one corrections); ``spb_weighted_gram`` = fp64 SIMT kernels (small-K variant below 33 inducing points).
"""

import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _problem(K, N, seed=0):
    rng = np.random.default_rng(seed)
    z = rng.uniform(-1.5, 1.5, size=(K, 3))
    x = rng.uniform(-1.7, 1.7, size=(N, 3))
    U = np.exp(-0.05 * ((x[:, None, :] - z[None, :, :]) ** 2).sum(-1)).astype(np.float32)  # [N, K] RBF like con_K
    w = (rng.uniform(0, 1, size=N) ** 4).astype(np.float32)
    w[rng.uniform(size=N) < 0.3] = 0.0
    X = rng.normal(size=(N, 3)).astype(np.float32)
    return U, w, X


def _device_inputs(U, w, X):
    import torch

    N, K = U.shape
    ldn = ((N + 1023) // 1024) * 1024
    dev = torch.device("cuda", 0)
    UT = torch.full((K, ldn), 7.0, dtype=torch.float32, device=dev)  # pad columns hold junk on purpose
    UT[:, :N] = torch.from_numpy(np.ascontiguousarray(U.T)).to(dev)
    wd = torch.zeros((ldn,), dtype=torch.float32, device=dev)
    wd[:N] = torch.from_numpy(w).to(dev)
    X3 = torch.zeros((3, ldn), dtype=torch.float32, device=dev)
    X3[:, :N] = torch.from_numpy(np.ascontiguousarray(X.T)).to(dev)
    return UT, wd, X3, ldn


@pytest.mark.parametrize("K,N", [(15, 5000), (64, 7000), (130, 9001), (200, 30011), (257, 4100), (500, 20000)])
def test_gram_tc_matches_float64(K, N):
    import torch

    from spateo_release_b200 import _capi
    from spateo_release_b200._capi import check, ptr

    lib = _capi.load_library()
    U, w, X = _problem(K, N)
    UT, wd, X3, ldn = _device_inputs(U, w, X)
    st = _capi.current_stream_ptr()
    hi, lo = torch.empty_like(UT), torch.empty_like(UT)
    mean = torch.empty((K,), dtype=torch.float32, device=UT.device)
    check(lib.spb_gram_center(ptr(UT), ldn, N, K, ptr(mean), ptr(hi), ptr(lo), st), "center")
    Bhi = torch.empty((K + 4, ldn), dtype=torch.float32, device=UT.device)
    Blo = torch.empty_like(Bhi)
    sums = torch.empty((4,), dtype=torch.float64, device=UT.device)
    need = C.c_int64(0)
    check(lib.spb_gram_tc_scratch_floats(K, 3, N, C.byref(need)), "plan")
    scratch = torch.empty((need.value,), dtype=torch.float32, device=UT.device)
    G = torch.full((K, K), -1.0, dtype=torch.float64, device=UT.device)
    R = torch.full((K, 3), -1.0, dtype=torch.float64, device=UT.device)
    for _ in range(2):  # twice: the scratch slabs are fully rewritten by every call
        check(lib.spb_gram_prepare(ptr(UT), ldn, N, K, ptr(mean), ptr(wd), ptr(X3), ldn, 3, ptr(Bhi), ptr(Blo), ptr(sums), st),
              "prepare")
        check(lib.spb_gram_tc(ptr(hi), ptr(lo), ptr(Bhi), ptr(Blo), ldn, N, K, 3, ptr(mean), ptr(sums), ptr(scratch),
                              scratch.numel(), ptr(G), ptr(R), st), "gram_tc")
    torch.cuda.synchronize()
    U64, w64, X64 = U.astype(np.float64), w.astype(np.float64), X.astype(np.float64)
    wantG = U64.T @ (U64 * w64[:, None])
    wantR = U64.T @ X64
    G, R = G.cpu().numpy(), R.cpu().numpy()
    eG = np.abs(G - wantG).max() / np.abs(wantG).max()
    # U^T X sums signed terms: scale by the sum of magnitudes
    eR = np.abs(R - wantR).max() / (np.abs(U64).T @ np.abs(X64)).max()
    print(f"\n[gram_tc K={K} N={N}] UtWU rel err {eG:.2e}  UtX rel err {eR:.2e}  asym {np.abs(G - G.T).max():.1e}")
    assert eG < 5e-7 and eR < 5e-7
    assert np.array_equal(G, G.T)


@pytest.mark.parametrize("K,N", [(3, 900), (15, 5000), (32, 7000), (40, 3000)])
def test_weighted_gram_fp64_kernels(K, N):
    import torch

    from spateo_release_b200 import _capi
    from spateo_release_b200._capi import check, ptr

    lib = _capi.load_library()
    U, w, X = _problem(K, N, seed=1)
    UT, wd, X3, ldn = _device_inputs(U, w, X)
    G = torch.empty((K, K), dtype=torch.float64, device=UT.device)
    R = torch.empty((K, 3), dtype=torch.float64, device=UT.device)
    check(lib.spb_weighted_gram(ptr(UT), ldn, N, K, ptr(wd), ptr(X3), ptr(G), ptr(R), _capi.current_stream_ptr()), "gram")
    torch.cuda.synchronize()
    U64, X64 = U.astype(np.float64), X.astype(np.float64)
    # the kernels round w * u to fp32 (like the reference's fp32 product) and mirror off-diagonal tiles: 1e-7 relative
    want = U64.T @ (U64 * w.astype(np.float64)[:, None])
    assert np.abs(G.cpu().numpy() - want).max() < 2e-7 * np.abs(want).max()
    assert np.abs(R.cpu().numpy() - U64.T @ X64).max() < 1e-11 * (np.abs(U64).T @ np.abs(X64)).max()
