"""Writes tests/golden/reference_checks.npz from the UNMODIFIED reference (oracle/ref_import.py): what the reference's own
postprocess and pad_image / pre_img return on fixed seeded inputs, so that tests/test_oracle_golden.py and
tests/test_preproc_oracle.py compare the oracles against it without the reference tree.

    python -m oracle.make_golden_reference_checks

Decode: the reference keypoints of O.make_decode_maps(2, 17, 999), crop i with org_wh (200 + i, 300 + i).
Pre-processing: 12 seeded boxes on P.make_frame(200, 260, 5) (boxes that are empty after clipping are skipped, as the test
did); per box the padded canvas, its (left, top), pre_img's org size and a seeded sample of 4096 values of pre_img's float
output (the full [1, 3, 256, 192] tensors of all boxes would be 7 MB).  The first PRE_FULL boxes also store that output whole and
exactly: per channel it takes at most 256 distinct values (a normalised uint8 image), kept as a value table and a uint8 index."""
import os

import numpy as np

from oracle import preproc_oracle as P, ref_import, vitpose_oracle as O

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_checks.npz")
PRE_SAMPLES = 4096
PRE_FULL = 3


def pack_exact(x):
    """[1, 3, H, W] float32 -> (per-channel value table [3, 256], uint8 index [3, H, W]) with table[c][index[c]] == x[0, c]."""
    x = np.asarray(x, np.float32)[0]
    table = np.zeros((3, 256), np.float32)
    index = np.zeros(x.shape, np.uint8)
    for c in range(3):
        vals, inv = np.unique(x[c], return_inverse=True)
        assert len(vals) <= 256
        table[c, :len(vals)] = vals
        index[c] = inv.reshape(x.shape[1:])
    return table, index


def unpack_exact(table, index):
    return np.stack([table[c][index[c]] for c in range(3)], 0)[None]


def pre_boxes():
    """The boxes of the pre-processing check, with their clipped padded extents (same draws as the original live test)."""
    rs = np.random.RandomState(2)
    out = []
    for _ in range(12):
        x0, y0 = rs.randint(-20, 240), rs.randint(-20, 180)
        box = np.array([x0, y0, x0 + rs.randint(1, 150), y0 + rs.randint(1, 150)])
        bx0, by0, bx1, by1 = P.padded_box(box, 200, 260)
        if bx1 <= bx0 or by1 <= by0:
            continue
        out.append((box, (bx0, by0, bx1, by1)))
    return out


def pre_sample_index(i):
    return np.random.RandomState(100 + i).randint(0, 3 * 256 * 192, size=PRE_SAMPLES)


def main():
    ns = ref_import.load()
    maps = O.make_decode_maps(2, 17, 999)
    dec = np.concatenate([ref_import.postprocess(ns, maps[i:i + 1], 200 + i, 300 + i) for i in range(2)], 0).astype(np.float64)

    inf = ref_import.load_vitinference()
    frame = P.make_frame(200, 260, 5)
    stub = type("S", (), {"target_size": (192, 256)})()
    out = {"decode_kpts": dec}
    boxes, lefttop, org, samples = [], [], [], []
    for i, (box, (bx0, by0, bx1, by1)) in enumerate(pre_boxes()):
        padded, (left, top) = inf.pad_image(frame[by0:by1, bx0:bx1], 3 / 4)
        x, org_h, org_w = inf.VitInference.pre_img(stub, padded)
        out[f"canvas_{i}"] = np.ascontiguousarray(padded)
        boxes.append(box)
        lefttop.append((left, top))
        org.append((org_h, org_w))
        samples.append(np.asarray(x, np.float32).reshape(-1)[pre_sample_index(i)])
        if i < PRE_FULL:
            out[f"pre_x_table_{i}"], out[f"pre_x_index_{i}"] = pack_exact(x)
            assert np.array_equal(unpack_exact(out[f"pre_x_table_{i}"], out[f"pre_x_index_{i}"]), np.asarray(x, np.float32))
    out.update(pre_boxes=np.array(boxes, np.int64), pre_left_top=np.array(lefttop, np.int64), pre_org_hw=np.array(org, np.int64),
               pre_x_sample=np.array(samples, np.float32))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
