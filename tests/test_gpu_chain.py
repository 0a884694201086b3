"""GPU: chain alignment drivers (morpho_align_transformation / apply, sharded variant, checkpoint + resume)."""

import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _chain(n_slices=4, n=2500, g=30, seed=0):
    """Slices that are rigid copies (plus jitter, re-sampled counts) of one base slice."""
    import pandas as pd

    from spateo_release_b200.anndata_lite import AnnDataLite

    rng = np.random.default_rng(seed)
    base = rng.uniform(0, 100, size=(n, 2))
    W = rng.normal(size=(2, g))
    phi = rng.uniform(0, 2 * np.pi, size=g)
    var = pd.DataFrame(index=[f"g{i}" for i in range(g)])
    out, poses = [], []
    for k in range(n_slices):
        th, sh = 0.25 * k, np.array([3.0 * k, -2.0 * k])
        perm = rng.permutation(n)
        c = base[perm]
        lam = np.exp(np.sin(c @ W / 30.0 + phi))
        X = rng.poisson(lam).astype(np.float32)
        R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
        raw = c @ R.T + sh + rng.normal(0, 0.2, size=c.shape)
        out.append(AnnDataLite(X, var=var.copy(), obsm={"spatial": raw, "truth": c}))
        poses.append((R, sh))
    return out, poses


def test_transformation_chain_recovers_poses(tmp_path):
    import spateo_release_b200 as st

    models, poses = _chain()
    np.random.seed(0)
    tdir = os.path.join(tmp_path, "tr")
    tr = st.align.morpho_align_transformation(models, device="0", verbose=False, SVI_mode=False, max_iter=100,
                                              save_transformation=True, transformation_path=tdir)
    assert len(tr) == 3 and all(set(t) == {"Rotation", "Translation"} for t in tr)
    assert sorted(os.listdir(tdir)) == [f"transformation_{i}.npy" for i in range(3)]
    st.align.morpho_align_apply_transformation(models, transformation=tr)
    ref = np.asarray(models[0].obsm["align_spatial"])
    # every slice, mapped through the composed chain, lands on slice 0's frame: compare via the known ground truth
    R0, s0 = poses[0]
    for m in models[1:]:
        want = np.asarray(m.obsm["truth"]) @ R0.T + s0
        err = np.abs(np.asarray(m.obsm["align_spatial"]) - want)
        assert err.mean() < 1.0 and err.max() < 4.0, (err.mean(), err.max())  # jitter 0.2 per link, domain 100
    assert np.allclose(ref, models[0].obsm["spatial"])
    # transformations can be re-read from the checkpoint directory
    models2, _ = _chain()
    st.align.morpho_align_apply_transformation(models2, transformation=None, transformation_path=tdir)
    assert np.allclose(models2[2].obsm["align_spatial"], models[2].obsm["align_spatial"])


def test_sharded_chain_single_process_equals_serial():
    import spateo_release_b200 as st

    models, _ = _chain(n_slices=3, n=1800)
    np.random.seed(0)
    tr_serial = st.align.morpho_align_transformation([m.copy() for m in models], device="0", verbose=False, SVI_mode=False, max_iter=60)
    np.random.seed(0)
    out, tr = st.align.morpho_align_chain_sharded([m.copy() for m in models], device="cuda:0", verbose=False, SVI_mode=False,
                                                  max_iter=60, dtype="float32")
    for a, b in zip(tr_serial, tr):
        assert np.allclose(a["Rotation"], b["Rotation"], atol=1e-6) and np.allclose(a["Translation"], b["Translation"], atol=1e-4)
    assert "align_spatial" in out[2].obsm


def test_morpho_align_ref_carries_the_field_to_the_full_slices():
    """morpho_align_ref (morpho_alignment.py:318-454): align random sub-samples, then place every cell of the full slices
    with BA_transform; the full slice must land where a direct alignment puts it."""
    import spateo_release_b200 as st

    models, poses = _chain(n_slices=2, n=3000)
    np.random.seed(0)
    full, small, pis, pis_ref = st.align.morpho_align_ref(models, n_sampling=1500, device="0", verbose=False, SVI_mode=False,
                                                         max_iter=100, mode="SN-S")
    assert len(full) == 2 and len(small) == 2 and small[1].shape[0] == 1500
    assert pis_ref[0].shape == (1500, 1500)
    for key in ("align_spatial", "align_spatial_rigid", "align_spatial_nonrigid"):
        assert full[1].obsm[key].shape == (3000, 2) and small[1].obsm[key].shape == (1500, 2)
    assert "VecFld_morpho" in full[1].uns and "iter_spatial" in small[1].uns
    # slice 0 is untouched; slice 1 is mapped back onto slice 0's frame: compare with the ground-truth positions
    assert np.array_equal(full[0].obsm["align_spatial"], models[0].obsm["spatial"])
    R0, s0 = poses[0]
    truth_in_frame0 = full[1].obsm["truth"] @ R0.T + s0
    err = np.linalg.norm(full[1].obsm["align_spatial"] - truth_in_frame0, axis=1)
    assert err.mean() < 1.0, err.mean()
    with pytest.raises(NotImplementedError):
        st.align.morpho_align_ref(models, sampling_method="trn", device="0")


def test_pipelined_chain_equals_serial_chain():
    """align_chain_pipelined (next pair prepared on a second stream under the current pair's EM, iterations replayed from
    CUDA graphs) gives the transformations of the serial driver and places every slice on slice 0's frame."""
    import spateo_release_b200 as st

    models, poses = _chain(n_slices=4, n=2200)
    kw = dict(verbose=False, SVI_mode=False, max_iter=80)
    np.random.seed(0)
    tr_serial = st.align.morpho_align_transformation([m.copy() for m in models], device="0", **kw)
    np.random.seed(0)
    stats = {}
    mine = [m.copy() for m in models]
    placed, tr = st.align.align_chain_pipelined(lambda k: mine[k], 4, device="0", stats=stats, **kw)
    assert stats["pairs"] == [0, 1, 2] and len(stats["seconds_per_pair"]) == 3 and stats["kernel_launches"] > 0
    for a, b in zip(tr_serial, tr):
        assert np.allclose(a["Rotation"], b["Rotation"], atol=1e-5) and np.allclose(a["Translation"], b["Translation"], atol=1e-3)
    R0, s0 = poses[0]
    for k in (1, 2, 3):
        want = np.asarray(placed[k].obsm["truth"]) @ R0.T + s0
        assert np.abs(np.asarray(placed[k].obsm["align_spatial"]) - want).mean() < 1.0
    assert np.allclose(placed[0].obsm["align_spatial"], models[0].obsm["spatial"])


def test_pipelined_chain_without_room_for_two_pairs(monkeypatch):
    """When the device cannot hold the next pair beside the current one (two 125k-cell cost matrices on an 80 GB GPU),
    align_chain_pipelined frees the current pair before preparing the next: same transformations as the serial driver."""
    import spateo_release_b200 as st
    from spateo_release_b200.alignment import distributed

    asked = []
    monkeypatch.setattr(distributed, "_room_for_next_pair", lambda dev, need: asked.append(need) or False)
    models, _ = _chain(n_slices=4, n=2200)
    kw = dict(verbose=False, SVI_mode=False, max_iter=80)
    np.random.seed(0)
    tr_serial = st.align.morpho_align_transformation([m.copy() for m in models], device="0", **kw)
    np.random.seed(0)
    mine = [m.copy() for m in models]
    placed, tr = st.align.align_chain_pipelined(lambda k: mine[k], 4, device="0", **kw)
    assert len(asked) == 2 and all(n > 4 * 2200 * 2200 for n in asked)
    for a, b in zip(tr_serial, tr):
        assert np.allclose(a["Rotation"], b["Rotation"], atol=1e-5) and np.allclose(a["Translation"], b["Translation"], atol=1e-3)
    assert sorted(placed) == [0, 1, 2, 3]


def test_gather_transformations_under_nccl_resolves_index_strings():
    """With an NCCL process group the slab must live on the CUDA device even when the package-style device string ("0") or
    None is passed (round-1 advisor finding); single rank, so no second GPU is needed."""
    import socket

    import torch
    import torch.distributed as dist

    from spateo_release_b200.alignment.distributed import gather_transformations

    if dist.is_initialized():
        pytest.skip("a process group already exists in this process")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK="0", WORLD_SIZE="1")
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    try:
        local = {p: {"Rotation": np.eye(2) * (p + 1), "Translation": np.array([p, -p], dtype=float)} for p in range(3)}
        for dev in ("0", None, "cuda:0"):
            out = gather_transformations(local, 3, device=dev)
            assert [float(t["Rotation"][0, 0]) for t in out] == [1.0, 2.0, 3.0]
            assert np.allclose(out[2]["Translation"], [2.0, -2.0])
    finally:
        dist.destroy_process_group()


def _rel_coords(a, b):
    return float(np.abs(np.asarray(a, dtype=np.float64) - b).max() / np.abs(b).max())


@pytest.mark.parametrize("mode", ["SN-S", "SN-N"])
def test_morpho_align_driver_matches_reference_driver(golden, mode):
    """``st.align.morpho_align`` (serial chain: pair i+1 starts from pair i's aligned coordinates, morpho_alignment.py:66-111)
    against the UNMODIFIED reference driver on the same four slices (tests/golden/make_golden_drivers.py): every slice's
    rigid / non-rigid / final placement within 1e-3 of the coordinate range, same uns keys, same pi shapes."""
    import spateo_release_b200 as st
    from driver_helpers import KW, models_from_golden

    g = golden("drivers")
    tag = mode.replace("-", "")
    np.random.seed(0)
    aligned, pis = st.align.morpho_align(models_from_golden(g), mode=mode, device="0", verbose=False, **KW)
    assert [tuple(p.shape) for p in pis] == [tuple(s) for s in g[f"{tag}_pi_shapes"]]
    assert sorted(aligned[1].uns.keys()) == list(g[f"{tag}_uns_keys_1"])
    for k in range(4):
        for key in ("align_spatial", "align_spatial_rigid", "align_spatial_nonrigid"):
            err = _rel_coords(aligned[k].obsm[key], g[f"{tag}_{k}_{key}"])
            assert err < 1e-3, (k, key, err)
    sums = np.array([float(np.asarray(p, dtype=np.float64).sum()) for p in pis])
    assert np.allclose(sums, g[f"{tag}_pi_sums"], rtol=2e-2)


def test_transformation_chain_matches_reference_driver(golden):
    """``morpho_align_transformation`` + ``morpho_align_apply_transformation`` (independent pairs on raw coordinates, composed;
    morpho_alignment.py:181-217, 284-303) against the reference driver's links and placements."""
    import spateo_release_b200 as st
    from driver_helpers import KW, models_from_golden

    g = golden("drivers")
    ms = models_from_golden(g)
    np.random.seed(0)
    tr = st.align.morpho_align_transformation(ms, device="0", verbose=False, **KW)
    assert len(tr) == 3
    for i, t in enumerate(tr):
        assert np.abs(np.asarray(t["Rotation"]) - g[f"tr{i}_Rotation"]).max() < 1e-4, i
        assert np.abs(np.asarray(t["Translation"]) - g[f"tr{i}_Translation"]).max() < 1e-3 * np.abs(g["in0_spatial"]).max(), i
    placed = st.align.morpho_align_apply_transformation(ms, transformation=tr, verbose=False)
    for k in range(4):
        assert _rel_coords(placed[k].obsm["align_spatial"], g[f"placed{k}"]) < 1e-3, k
