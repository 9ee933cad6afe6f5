"""Host side of the device detection backend: the per-chip table `ops.detect_post` reads, the 64-bit order key and the
order it induces, and `inference.aggregate`'s refusal of mixed backends."""
import numpy as np
import pytest

from sniper_b200 import inference


def test_chip_table_hand_cases():
    # a landscape and a portrait image; chips touching each image border, and one touching none
    roidb = [dict(width=640, height=480, inference_crops=np.array([[0, 0, 640, 480]])),
             dict(width=300, height=500, inference_crops=np.array([[0.25, 40.0, 200.0, 300.0],      # left border
                                                                    [50.0, 0.0, 250.0, 310.5],       # top
                                                                    [100.0, 60.0, 299.75, 400.0],    # right
                                                                    [20.0, 180.0, 260.0, 500.0],     # bottom
                                                                    [32.0, 48.0, 200.5, 320.25]]))]  # none
    t = inference.chip_table(roidb, [0, 1, 1, 1, 1, 1], [0, 0, 1, 2, 3, 4], True, (16, 90))
    assert t.dtype == np.float64 and t.shape == (6, inference.CHIP_COLS)
    assert t[0].tolist() == [0, 0, 0, 0, 640, 480, 640, 480, 1, 16, 90, 0]
    assert t[1].tolist() == [1, 0, 0.25, 40, 200, 300, 300, 500, 1, 16, 90, 0]
    assert t[5].tolist() == [1, 4, 32, 48, 200.5, 320.25, 300, 500, 1, 16, 90, 0]
    # which borders the kernel's check_valid will test: a chip border that is not an image border
    tests = [(bool(r[2] >= 0.5), bool(r[3] >= 0.5), bool(r[4] < r[6] - 0.5), bool(r[5] < r[7] - 0.5)) for r in t]
    assert tests == [(False, False, False, False), (False, True, True, True), (True, False, True, True),
                     (True, True, False, True), (True, True, True, False), (True, True, True, True)]
    # no pruning, open valid range
    t = inference.chip_table(roidb, [1], [2], False, (-1, 40))
    assert t[0, 8] == 0 and t[0, 9] == -1 and t[0, 10] == 40


def test_chip_table_marks_repeated_chips_and_refuses_ids_outside_the_key():
    roidb = [dict(width=64, height=64, inference_crops=np.array([[0, 0, 64, 64], [0, 0, 32, 32]]))]
    seen = set()
    t = inference.chip_table(roidb, [0, 0, 0], [0, 1, 0], False, (-1, -1), seen)
    assert t[:, 0].tolist() == [0, 0, -1] and seen == {(0, 0), (0, 1)}
    t = inference.chip_table(roidb, [0, 0], [1, 1], False, (-1, -1), seen)      # the iterator's padding of a last batch
    assert t[:, 0].tolist() == [-1, -1]
    big = [dict(width=8, height=8, inference_crops=np.zeros((1 << 14) + 1, dtype=object))]
    with pytest.raises(ValueError):
        inference.chip_table(big, [0], [1 << 14], False, (-1, -1))


def test_key_round_trip_and_field_order():
    rng = np.random.RandomState(0)
    f = [rng.randint(0, 1 << b, 1000) for b in (19, 10, 4, 14, 16)]
    key = inference.pack_key(*f)
    assert key.dtype == np.int64 and (key >= 0).all()
    for a, b in zip(inference.unpack_key(key), f):
        assert np.array_equal(a, b)
    # the layout the kernel writes: image << 44 | class << 34 | scale << 30 | chip << 16 | roi
    assert int(inference.pack_key(3, 7, 2, 5, 9)) == (3 << 44) | (7 << 34) | (2 << 30) | (5 << 16) | 9
    # lexicographic in (image, class, scale, chip, roi)
    tup = sorted(zip(*[x.tolist() for x in f]))
    assert sorted(key.tolist()) == [int(inference.pack_key(*t)) for t in tup]


def test_key_order_is_the_stacking_order_of_aggregate():
    """Equal scores and disjoint boxes make `cpu_soft_nms` return its input order, so the host aggregation shows the
    order in which it stacked each (image, class) problem: scale, then chip, then row.  Sorting by key must give it."""
    rng = np.random.RandomState(1)
    K, n_img, n_scale = 4, 2, 3
    n_chips = [[1, 1], [2, 3], [3, 1]]                      # per scale, per image
    nested, rows, keys = [], [], []
    uid = 0
    for s in range(n_scale):
        per_cls = [[[np.zeros((0, 5), np.float32) for _ in range(n_chips[s][i])] for i in range(n_img)] for _ in range(K)]
        for i in range(n_img):
            for c in range(n_chips[s][i]):
                rois = np.sort(rng.choice(300, 4, replace=False))
                for j in range(1, K):
                    pick = rois[rng.rand(4) < 0.7]
                    d = np.zeros((len(pick), 5), np.float32)
                    for k, r in enumerate(pick):
                        d[k] = [100.0 * uid, 0, 100.0 * uid + 10, 10, 0.5]      # disjoint, the x1 identifies the row
                        rows.append(d[k].copy())
                        keys.append(int(inference.pack_key(i, j, s, c, r)))
                        uid += 1
                    per_cls[j][i][c] = d
        nested.append(per_cls)
    want = inference.aggregate(nested, [(-1, -1)] * n_scale, n_img, K, max_per_image=0, backend="host")
    rows, keys = np.array(rows), np.array(keys, np.int64)
    order = np.argsort(keys, kind="stable")
    rows, keys = rows[order], keys[order]
    img, cls = inference.unpack_key(keys)[:2]
    n = 0
    for i in range(n_img):
        for j in range(1, K):
            got = rows[(img == i) & (cls == j)]
            assert np.array_equal(got, want[j][i]), (i, j)
            n += len(got)
    assert n == len(rows) > 30


def test_aggregate_refuses_mixed_backends():
    dev = inference.DeviceDetections.__new__(inference.DeviceDetections)        # no buffer needed to be refused
    lists = [[[np.zeros((0, 5), np.float32)]] for _ in range(3)]
    with pytest.raises(TypeError, match="same backend"):
        inference.aggregate([lists, dev], [(-1, -1), (-1, -1)], 1, 3, backend="host")
    with pytest.raises(TypeError, match="same backend"):
        inference.aggregate([dev, lists], [(-1, -1), (-1, -1)], 1, 3, backend="host")
