"""CPU: the decode oracles at the keypoint counts the C ABI promises but the other fixtures never use (K = 1, 2, 32, 33, 144)
against the outputs of the UNMODIFIED reference committed in tests/golden/decode_k_edges.npz (oracle/make_golden_k_edges.py).

One case has no reference output: keypoints_from_heatmaps(use_udp=True) on an [N > 1, 1, 64, 48] array raises in the reference
(post_dark_udp's `.squeeze()`, top_down_eval.py:414, drops the K axis).  The fixture records that raise as a flag; the Python
wrapper raises there too, and the C entry points decode the case with the formula's intended shape (O.decode_maps(wrap="batch"),
checked on the GPU in tests/test_gpu_limits.py)."""
import os

import numpy as np
import pytest

from oracle import decode_modes_oracle as M, vitpose_oracle as O
from oracle.make_golden_k_edges import COMBOS, KS, MODE_KS, N, centre_scale_of, org_of, seed_of


@pytest.fixture(scope="module")
def golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "decode_k_edges.npz"))
    assert tuple(int(v) for v in g["meta"]) == (N, *KS)
    return g


def _assert_close(kp, ref, K):
    """scores bit-exact; coordinates of real peaks within 1e-3 px, sentinel / flat / noise maps relatively (test_oracle_golden)"""
    assert np.array_equal(kp[..., 2], ref[..., 2])
    err = np.abs(kp[..., :2] - ref[..., :2])
    well = np.isin((np.arange(N * K) % 10).reshape(N, K), [0, 1, 2, 3, 5, 7])
    assert err[well].max() < 1e-3
    assert np.all(err[~well] <= 1e-3 + 1e-3 * np.abs(ref[..., :2][~well]))


@pytest.mark.parametrize("K", KS)
def test_per_crop_decode_matches_reference(golden, K):
    """VitInference.postprocess, one reference call per crop: what vpb_decode(wrap_batch = 0) and the engine's crop and frame
    calls compute."""
    maps = O.make_decode_maps(N, K, seed_of(K))
    kp, idx = O.decode_maps(maps, org_of(K), wrap="crop")
    assert np.array_equal(idx, np.argmax(maps.reshape(N, K, -1), -1))
    _assert_close(kp, golden[f"crop_{K}_kpts"], K)


@pytest.mark.parametrize("K", KS)
def test_batched_decode_matches_reference_or_raises(golden, K):
    """One reference call on the [N,K] array (vpb_decode(wrap_batch = 1)): it runs for K >= 2 and raises for K = 1."""
    assert int(golden[f"batch_{K}_raises"]) == (K == 1)
    if K == 1:
        return
    kp, _ = O.decode_maps(O.make_decode_maps(N, K, seed_of(K)), org_of(K), wrap="batch")
    _assert_close(kp, golden[f"batch_{K}_kpts"], K)


def test_wrap_matters_at_one_keypoint():
    """At K = 1 the sentinel's "previous map" is the map itself per crop and the previous crop's map per batch: the two
    readings must differ on this fixture's maps, or the wrap_batch = 1 checks at K = 1 would not test anything."""
    maps = O.make_decode_maps(N, 1, seed_of(1))
    kinds = np.arange(N) % 10
    assert np.isin(kinds, [4, 6]).any() and (maps.reshape(N, -1).max(-1) <= 0)[1:].any()
    a, _ = O.decode_maps(maps, org_of(1), wrap="crop")
    b, _ = O.decode_maps(maps, org_of(1), wrap="batch")
    assert not np.array_equal(a, b)


@pytest.mark.parametrize("pp,udp", COMBOS)
@pytest.mark.parametrize("K", MODE_KS)
def test_decode_modes_match_reference(golden, K, pp, udp):
    key = f"k{K}_{pp}_{'udp' if udp else 'std'}"
    raises = int(golden[key + "_raises"])
    assert raises == (K == 1 and udp)
    if raises:
        return
    c, s = centre_scale_of(K)
    preds, maxvals, _ = M.keypoints_from_heatmaps(O.make_decode_maps(N, K, seed_of(K)), c, s, post_process=pp, use_udp=udp)
    assert np.array_equal(maxvals, golden[key + "_maxvals"], equal_nan=True)
    ref = golden[key + "_preds"]
    if pp in (None, "default", "megvii") and not udp:
        assert np.array_equal(preds, ref, equal_nan=True)
    else:
        assert np.array_equal(np.isnan(preds), np.isnan(ref)) and np.nanmax(np.abs(preds - ref)) < 1e-3


def test_combined_target_one_keypoint_matches_reference(golden):
    """CombinedTarget (mode 5) with K = 1, one reference call per crop: bit-exact, sentinels included."""
    cmaps = M.make_combined_maps(N, 1, seed_of(1) + 3)
    c, s = centre_scale_of(1)
    for n in range(N):
        p, mv, _ = M.combined_target(cmaps[n:n + 1], c[n:n + 1], s[n:n + 1], 11)
        assert np.array_equal(mv[0], golden["comb_maxvals"][n], equal_nan=True), n
        assert np.array_equal(p[0], golden["comb_preds"][n], equal_nan=True), n


def test_python_wrapper_raises_like_the_reference():
    """keypoints_from_heatmaps(use_udp=True) on one-keypoint maps: ValueError for N > 1 (before any device work), as the
    reference raises."""
    from easy_vitpose_b200 import keypoints_from_heatmaps
    c, s = centre_scale_of(1)
    for n in (2, N):
        with pytest.raises(ValueError, match="K=1"):
            keypoints_from_heatmaps(np.zeros((n, 1, 64, 48), np.float32), c[:n], s[:n], use_udp=True)
        with pytest.raises(ValueError, match="K=1"):
            keypoints_from_heatmaps(np.zeros((n, 1, 64, 48), np.float32), c[:n], s[:n], unbiased=True, use_udp=True)


def test_live_reference_raises_at_one_keypoint():
    """The flag in the fixture against the reference itself, where the reference tree is present."""
    import warnings

    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference tree not present")
    ns = ref_import.load()
    maps = O.make_decode_maps(N, 1, seed_of(1))
    org = org_of(1)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(ValueError):
            ns.keypoints_from_heatmaps(maps.copy(), np.stack([org[:, 0] // 2, org[:, 1] // 2], 1), org.astype(np.int64),
                                       unbiased=True, use_udp=True)
        ns.keypoints_from_heatmaps(maps[:1].copy(), org[:1] // 2, org[:1].astype(np.int64), unbiased=True, use_udp=True)
