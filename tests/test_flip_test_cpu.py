"""CPU: the host side of the flip test -- dataset flip pairs, the keypoint permutation the engine receives, and the index
maps of the two mirrored patch gathers (pointwise.cuh: patch_im2col, preprocess.cuh: frame_to_patch_rows) restated in
numpy against the oracle's im2col of the flipped crops."""
import numpy as np
import pytest

from oracle import decode_modes_oracle as DM, vitpose_oracle as O


def test_flip_pairs_for_datasets():
    from easy_vitpose_b200 import COCO_FLIP_PAIRS, flip_pairs_for
    assert flip_pairs_for("coco") == [tuple(p) for p in DM.COCO_FLIP_PAIRS]     # the oracle's copy of datasets/COCO.py:114
    assert list(COCO_FLIP_PAIRS) == flip_pairs_for("coco")
    for ds in ("ap10k", "wholebody", "coco_25", "mpii", None):
        with pytest.raises(ValueError):
            flip_pairs_for(ds)
    assert flip_pairs_for("ap10k", [[0, 1], (2, 3)]) == [(0, 1), (2, 3)]
    assert flip_pairs_for("coco", [(5, 6)]) == [(5, 6)]


@pytest.mark.parametrize("pairs", [DM.COCO_FLIP_PAIRS, [(0, 1), (1, 2)], [(3, 5), (5, 3), (0, 4)]])
def test_sequential_permutation_equals_reference_loop(pairs):
    """The engine reads heatmap perm[k] of the mirrored crop for keypoint k; the permutation is built pair by pair, a later
    pair overriding an earlier one, like flip_back's loop -- also for overlapping pairs."""
    from easy_vitpose_b200 import ViTPose
    K = 17
    rs = np.random.RandomState(5)
    hm = rs.standard_normal((3, K, 64, 48)).astype(np.float32)
    perm = ViTPose.flip_permutation(K, pairs)
    for shift in (False, True):
        want = DM.flip_back(hm, pairs, shift)
        xs = np.arange(48)
        src_x = 47 - (np.maximum(xs - 1, 0) if shift else xs)
        got = hm[:, perm][..., src_x]
        assert np.array_equal(got, want)


def _mirrored_patch_im2col(x: np.ndarray) -> np.ndarray:
    """patch_im2col's mirrored mode as the kernel indexes it: thread (b, c, y', xc) covers image columns xx = 8 xc - 2 + j,
    reads the source pair at 190 - xx and swaps its halves."""
    B = x.shape[0]
    rows = np.zeros((B, 16, 12, 768), np.float32)
    for yp in range(256):
        y = yp - 2
        if y < 0:
            continue
        py, ky = yp >> 4, yp & 15
        for xc in range(24):
            px, kx0 = xc >> 1, (xc & 1) * 8
            for j in range(0, 8, 2):
                xx = xc * 8 - 2 + j
                if 0 <= xx < 192:
                    pair = x[:, :, y, 190 - xx:192 - xx]
                    for c in range(3):
                        rows[:, py, px, c * 256 + ky * 16 + kx0 + j] = pair[:, c, 1]
                        rows[:, py, px, c * 256 + ky * 16 + kx0 + j + 1] = pair[:, c, 0]
    return rows.reshape(B, 192, 768)


def test_mirrored_patch_gather_index_map():
    x = O.make_crops(2, 31)
    assert np.array_equal(_mirrored_patch_im2col(x), O.patch_rows(np.ascontiguousarray(np.flip(x, 3))))


def test_mirrored_frame_tile_index_map():
    """frame_to_patch_rows: a mirrored CTA stores crop pixel dx at tile column 2 + (191 - dx); the unchanged phase 2 then reads
    tile[c][ky][16 px + kx].  That must be the im2col of the mirrored crop."""
    x = O.make_crops(1, 32)[0]
    want = O.patch_rows(np.ascontiguousarray(np.flip(x, 2))[None])[0].reshape(16, 12, 3, 16, 16)
    for py in range(16):
        tile = np.zeros((3, 16, 208), np.float32)
        for ky in range(16):
            dy = 16 * py - 2 + ky
            if dy >= 0:
                tile[:, ky, 2 + (191 - np.arange(192))] = x[:, dy, :]
        for px in range(12):
            assert np.array_equal(tile[:, :, 16 * px:16 * px + 16], want[py, px]), (py, px)
