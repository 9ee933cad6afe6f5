"""The batched device soft-NMS (csrc/nms.cu) on exact score ties: every case of tests/soft_nms_cases.py, each method in
one launch of a run's worth of (image, class) problems, against the host port (bit-identical to the reference's loop,
tests/test_soft_nms_cases_cpu.py) and the reference's own Cython when it is built.  Same rows in the same order and the
same counts; scores exact for linear and hard NMS, within 1 ulp for the Gaussian (a double exp on both sides: glibc on
the host, CUDA libm on the device).  Also `inference.aggregate` on nested lists with saturated and duplicated rows:
device and host back ends give the same all_boxes."""
import numpy as np
import pytest

import soft_nms_cases as C

pytestmark = pytest.mark.gpu

NUM_CLASSES, NUM_IMAGES = 80, 5           # a run's problems: one per (image, class), most of them empty


def _run_layout():
    """Problem slots of the cases among NUM_IMAGES * NUM_CLASSES problems; every other problem is empty."""
    rng = np.random.RandomState(11)
    slots = np.sort(rng.permutation(NUM_IMAGES * NUM_CLASSES)[:len(C.CASE_NAMES)])
    return dict(zip(slots.tolist(), C.CASE_NAMES))


@pytest.mark.parametrize("method,sigma,Nt", C.METHODS)
def test_every_case_in_one_launch(method, sigma, Nt):
    import torch
    from sniper_b200 import ops
    layout = _run_layout()
    P = NUM_IMAGES * NUM_CLASSES
    probs = [C.build(layout[p]) if p in layout else np.zeros((0, 5), np.float32) for p in range(P)]
    sizes = [len(d) for d in probs]
    offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    dets_np = np.concatenate(probs, 0)
    dets = torch.from_numpy(dets_np).cuda()
    out, counts = ops.soft_nms_batched(dets, torch.from_numpy(offsets).cuda(), sigma=sigma, Nt=Nt,
                                       threshold=float(C.THRESHOLD), method=method)
    out, counts = out.cpu().numpy(), counts.cpu().numpy()
    assert np.array_equal(dets.cpu().numpy(), dets_np), "dets was modified"
    assert counts.shape == (P,) and all(counts[p] == 0 for p in range(P) if sizes[p] == 0)
    ref = None
    try:
        ref = C.ref_cython()
    except pytest.skip.Exception:
        pass
    failed = []
    for p, name in layout.items():
        d = probs[p]
        got = out[offsets[p]:offsets[p] + counts[p]]
        try:
            C.assert_same_output(got, C.host_soft_nms(d, sigma, Nt, method), method, name + ": device vs host port")
            if ref is not None and len(d):
                C.assert_same_output(got, C.cython_soft_nms(ref, d, sigma, Nt, method), method,
                                     name + ": device vs Cython")
        except AssertionError as e:
            failed.append(str(e).splitlines()[0])
    assert not failed, "%d of %d cases differ (method %d): %s" % (len(failed), len(layout), method, failed)


def _tied_nested_lists(rng, num_scales, num_images, num_classes):
    """scale_cls_dets[s][j][i] = chips of [n,5] rows: 40 objects per (image, class) seen at every scale and, within a
    scale, by two or three overlapping chips that report some of the same detections again (exact duplicate rows);
    scores of a saturated softmax (10-30 % of the rows at exactly 1.0f).  Some hundred rows per problem: enough for
    the Gaussian's first rounds to remove rows and move later rows at 1.0 ahead of earlier ones."""
    out = []
    objs = {(j, i): C._clustered_boxes(rng, 40) for j in range(1, num_classes) for i in range(num_images)}
    for _s in range(num_scales):
        per_class = [[[] for _ in range(num_images)] for _ in range(num_classes)]
        for j in range(1, num_classes):
            for i in range(num_images):
                o = objs[(j, i)]
                m = int(rng.randint(100, 250))
                b = o[rng.randint(0, len(o), m)] + (rng.randn(m, 4) * 3.0).astype(np.float32)
                b = np.concatenate([np.minimum(b[:, :2], b[:, 2:]), np.maximum(b[:, :2], b[:, 2:])], 1)
                rows = np.concatenate([b, C._saturated(rng, m)[:, None]], 1).astype(np.float32)
                chips = [rows]
                for _c in range(int(rng.randint(1, 3))):
                    chips.append(rows[np.sort(rng.permutation(m)[:m // 3])].copy())
                per_class[j][i] = chips
        out.append(per_class)
    return out


def test_aggregate_device_equals_host_path_with_ties():
    """Tester.aggregate (lib/inference.py:152-230) on detections with exact ties -- rows at 1.0f and exact duplicates
    across scales and chips -- through the device launch and through the host cpu_soft_nms: the same all_boxes, after
    the MAX_PER_IMAGE cut."""
    from sniper_b200 import inference
    rng = np.random.RandomState(12)
    num_images, num_classes, max_per_image = 3, 6, 40
    valid_ranges = [(-1, -1)] * 3               # every row reaches the soft-NMS (the area filter has its own test)
    scale_cls_dets = _tied_nested_lists(rng, 3, num_images, num_classes)
    rows = np.concatenate([c for s in scale_cls_dets for j in s for i in j for c in i], 0)
    assert (rows[:, 4] == 1.0).sum() > 100 and len(np.unique(rows, axis=0)) < len(rows)
    dev = inference.aggregate(scale_cls_dets, valid_ranges, num_images, num_classes, max_per_image=max_per_image)
    hst = inference.aggregate(scale_cls_dets, valid_ranges, num_images, num_classes, max_per_image=max_per_image,
                              backend="host")
    n = 0
    for j in range(1, num_classes):
        for i in range(num_images):
            C.assert_same_output(dev[j][i], hst[j][i], 2, "class %d image %d" % (j, i))
            n += len(dev[j][i])
    # the cut bites: every image has more than max_per_image detections before it
    uncut = inference.aggregate(scale_cls_dets, valid_ranges, num_images, num_classes, max_per_image=0, backend="host")
    assert all(sum(len(uncut[j][i]) for j in range(1, num_classes)) > max_per_image for i in range(num_images))
    assert 0 < n < sum(len(uncut[j][i]) for j in range(1, num_classes) for i in range(num_images))
