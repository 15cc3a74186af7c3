"""CPU checks of the affine top-down crop: the oracle (oracle/affine_oracle.py) against the fixture the unmodified reference
wrote (tests/golden/affine_b_coco.npz, oracle/make_golden_affine.py) and against live cv2 / torchvision where installed,
topdown_args against the fixture, and the Python argument checks of the affine calls."""
import os
import zlib

import numpy as np
import pytest
import torch

from oracle import affine_oracle as A, preproc_oracle as P


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "affine_b_coco.npz"))


def _frames(g):
    return [P.make_frame(int(h), int(w), int(s)) for h, w, s in g["frames"]]


def test_oracle_matches_fixture(golden):
    g = golden
    frames = _frames(g)
    stored = dict(zip(g["crop_ids"].tolist(), g["crops"]))
    for i, box in enumerate(g["boxes"]):
        c, s = A.xywh2cs(box)
        assert np.array_equal(c, g["centers"][i]) and np.array_equal(s, g["scales"][i]), i
        rot = float(g["rot"][i])
        if g["builder"][i] == 0:
            m = A.udp_matrix(c, s, rot)
            assert m.dtype == np.float32
        else:
            pytest.importorskip("cv2")
            m = A.hrnet_matrix(c, s, rot)
            assert m.dtype == np.float64
        assert np.array_equal(m.astype(np.float64), g["mats"][i]), i
        img = A.warp_affine_u8(frames[g["frame_id"][i]], g["mats"][i])
        assert zlib.crc32(img.tobytes()) == int(g["crc"][i]), i
        if i in stored:
            assert np.array_equal(img, stored[i]), i
    # the fixture's wholly-outside boxes warp to black crops
    for i in (6, 11):
        assert A.warp_affine_u8(frames[g["frame_id"][i]], g["mats"][i]).max() == 0, i
    assert np.array_equal(g["cs_px"][:, 2:], g["scales"][g["fwd"]] * np.float32(200.0))


def _random_matrices(n=200, seed=11):
    """Rotations, up / down scaling, shears, crops partly or wholly outside the frame, and singular matrices."""
    rs = np.random.RandomState(seed)
    out = []
    for i in range(n):
        if i % 25 == 0:
            m = np.zeros((2, 3)) if i % 50 == 0 else np.array([[1.0, 2.0, rs.uniform(-50, 50)], [0.5, 1.0, rs.uniform(-50, 50)]])
        else:
            th = np.deg2rad(rs.uniform(-60, 60))
            k = np.exp(rs.uniform(-2.5, 2.5))
            sh = rs.uniform(-0.3, 0.3) if i % 3 == 0 else 0.0
            m = np.array([[k * np.cos(th), -k * np.sin(th) + sh, 0.0], [k * np.sin(th), k * np.cos(th), 0.0]])
            m[:, 2] = rs.uniform(-600, 400, 2)
        out.append(m.astype(np.float32) if i % 2 else m)
    return out


def test_oracle_matches_cv2_on_random_matrices():
    cv2 = pytest.importorskip("cv2")
    frame = P.make_frame(200, 260, 9)
    for i, m in enumerate(_random_matrices()):
        want = cv2.warpAffine(frame, m, (192, 256), flags=cv2.INTER_LINEAR)
        assert np.array_equal(A.warp_affine_u8(frame, m), want), i


def test_normalise_table_matches_torchvision():
    transforms = pytest.importorskip("torchvision.transforms")
    tf = transforms.Compose([transforms.ToTensor(), transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])])
    img = np.tile(np.arange(256, dtype=np.uint8)[None, :, None], (2, 1, 3))
    assert np.array_equal(tf(img).numpy()[:, 0, :], A.normalise_table())


def test_topdown_args_match_fixture(golden):
    from easy_vitpose_b200 import topdown_args
    from easy_vitpose_b200 import topdown as T
    g = golden
    fwd = g["fwd"]
    mats, centers, scales = topdown_args(g["boxes"][fwd])
    assert mats.dtype == np.float64 and centers.dtype == np.float32 and scales.dtype == np.float32
    assert np.array_equal(mats, g["mats"][fwd]) and np.array_equal(centers, g["centers"][fwd])
    assert np.array_equal(scales, g["cs_px"][:, 2:])
    for i in range(len(g["boxes"])):
        c, s = g["centers"][i], g["scales"][i]
        rot = float(g["rot"][i])
        if g["builder"][i] == 0:
            assert np.array_equal(T.udp_matrix(c, s, rot).astype(np.float64), g["mats"][i]), i
        else:                   # cv2.getAffineTransform solves the same system in its own order: a few ulp apart
            np.testing.assert_allclose(T.hrnet_matrix(c, s, rot), g["mats"][i], rtol=1e-12, atol=1e-12 * np.abs(g["mats"][i]).max())
    hr = [i for i in range(len(g["boxes"])) if g["builder"][i] == 1 and g["rot"][i] == 0]
    m_hr, _, _ = topdown_args(g["boxes"][hr], use_udp=False)
    np.testing.assert_allclose(m_hr, g["mats"][hr], rtol=1e-12, atol=1e-9)
    m0, c0, s0 = topdown_args(np.zeros((0, 4)))
    assert m0.shape == (0, 2, 3) and c0.shape == (0, 2) and s0.shape == (0, 2)


def test_affine_argument_checks():
    from easy_vitpose_b200 import ViTPose
    args = ViTPose._affine_args
    m = np.tile(np.array([[1.0, 0, 0], [0, 1, 0]]), (3, 1, 1))
    c, s = np.zeros((3, 2), np.float32), np.full((3, 2), 100, np.float32)
    counts, M, CS = args([m, m[:1]], [c, c[:1]], [s, s[:1]])
    assert counts == [3, 1] and M.shape == (4, 6) and M.dtype == torch.float64 and CS.shape == (4, 4) and CS.dtype == torch.float32
    assert torch.equal(CS[:, 2:], torch.full((4, 2), 100.0))
    counts, M, CS = args([m.reshape(3, 6)])
    assert counts == [3] and CS is None
    with pytest.raises(ValueError, match="expected"):
        args([m[:, :, :2]])
    with pytest.raises(ValueError, match="expected"):
        args([np.zeros(6)])
    bad = m.copy()
    bad[1, 0, 2] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        args([bad])
    args([bad], validate=False)
    with pytest.raises(ValueError, match="scales > 0"):
        args([m], [c], [np.array([[100, 100], [100, 0], [100, 100]], np.float32)])
    with pytest.raises(ValueError, match="scales > 0"):
        args([m], [np.array([[0, np.inf], [0, 0], [0, 0]])], [s])
    with pytest.raises(ValueError, match="3 matrices, 2 centres"):
        args([m], [c[:2]], [s])
    with pytest.raises(ValueError, match="centre arrays"):
        args([m, m], [c], [s])
    assert args([])[0] == []
