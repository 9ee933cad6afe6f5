"""The training roidb from disk (sniper_b200.load_data) and the image reader (host.imread), on the host.

  * byte for byte against the reference's own load_proposal_roidb / merge_roidb / filter_roidb /
    add_bbox_regression_targets (tests/golden/train_roidb_ref.npz, oracle/run_ref_train_roidb.py), both branches
    (GT only, and RPN proposals from the NMS cache) with every normalisation mode;
  * host.imread against PIL's own decode for RGB, grayscale, palette, RGBA and EXIF-rotated files;
  * a VOCdevkit and a COCO image set written with JPEG files: flip, merge, filter, and the iterator's pixels of a
    flipped entry."""
import os
import pickle
import sys
import types

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import train_data_fixture as TD  # noqa: E402
from sniper_b200 import host, load_data  # noqa: E402
from sniper_b200 import iterator as IT  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "train_roidb_ref.npz")
YEARS = ("2007", "2012")
ROW_KEYS = ("boxes", "gt_classes", "gt_overlaps", "max_classes", "max_overlaps", "bbox_targets")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _write_golden_devkit(g, root):
    """The oracle's devkit and proposal caches, from the fixture."""
    dk, pp = os.path.join(root, "VOCdevkit"), os.path.join(root, "proposals")
    os.makedirs(pp, exist_ok=True)
    for year in YEARS:
        vp = os.path.join(dk, "VOC" + year)
        for sub in ("Annotations", "ImageSets/Main", "JPEGImages"):
            os.makedirs(os.path.join(vp, sub), exist_ok=True)
        names = [str(n) for n in g["devkit_%s_names" % year]]
        with open(os.path.join(vp, "ImageSets", "Main", "trainval.txt"), "w") as f:
            f.write("".join(n + "\n" for n in names))
        for n, xml in zip(names, g["devkit_%s_xml" % year]):
            with open(os.path.join(vp, "Annotations", n + ".xml"), "w") as f:
                f.write(str(xml))
            open(os.path.join(vp, "JPEGImages", n + ".jpg"), "w").close()
        props = [g["props_%s_%d" % (year, i)] for i in range(len(names))]
        with open(os.path.join(pp, "PASCALVOC_%s_trainval_rpn_after_nms.pkl" % year), "wb") as f:
            pickle.dump([props, []], f, 2)
    return dk, pp


def _cfg(precomputed, agnostic):
    cfg = IT.default_config(dataset="pascal_voc")
    cfg.CLASS_AGNOSTIC = agnostic
    cfg.TRAIN.BBOX_NORMALIZATION_PRECOMPUTED = precomputed
    return cfg


@pytest.mark.parametrize("mode", ["gt", "rpn"])
@pytest.mark.parametrize("precomputed", [True, False])
@pytest.mark.parametrize("agnostic", [True, False])
def test_roidb_equals_reference(golden, tmp_path, mode, precomputed, agnostic):
    g = golden
    k = "%s_%s_%s" % (mode, "pre" if precomputed else "acc", "agnostic" if agnostic else "perclass")
    dk, pp = _write_golden_devkit(g, str(tmp_path))
    cfg = _cfg(precomputed, agnostic)
    roidbs = []
    for year in YEARS:
        roidb, imdb = load_data.load_proposal_roidb("PascalVOC", year + "_trainval", str(tmp_path), dk, flip=True,
                                                    proposal_path=pp, only_gt=mode == "gt", get_imdb=True, device="cpu")
        n = len(g["devkit_%s_names" % year])
        assert len(roidb) == 2 * n and imdb.num_images == n and len(imdb.image_set_index) == 2 * n
        for a, b in zip(roidb[:n], roidb[n:]):
            assert all(a[key] is b[key] for key in ("gt_classes", "gt_overlaps", "max_classes", "max_overlaps"))
            assert (a.get("proposal_scores") is b.get("proposal_scores")) and (mode == "gt") == ("proposal_scores" not in a)
        roidbs.append(roidb)
    roidb = load_data.filter_roidb(load_data.merge_roidb(roidbs), cfg)
    means, stds = load_data.add_bbox_regression_targets(roidb, cfg)
    assert [os.path.relpath(r["image"], dk) for r in roidb] == [str(s) for s in g[k + "_image"]]
    assert np.array_equal([r["flipped"] for r in roidb], g[k + "_flipped"])
    assert np.array_equal([[r["height"], r["width"]] for r in roidb], g[k + "_hw"])
    assert np.array_equal([len(r["boxes"]) for r in roidb], g[k + "_n"])
    for key in ROW_KEYS:
        got = np.concatenate([np.asarray(r[key]) for r in roidb])
        assert got.dtype == g[k + "_" + key].dtype and got.tobytes() == g[k + "_" + key].tobytes(), key
    assert means.tobytes() == g[k + "_means"].tobytes() and stds.tobytes() == g[k + "_stds"].tobytes()
    if mode == "rpn":       # the case the fixture was built for: a proposal equal to a GT box regresses to itself
        mo = np.concatenate([r["max_overlaps"] for r in roidb])
        assert (mo == 1).sum() > sum((r["gt_classes"] > 0).sum() for r in roidb)


# ------------------------------------------------------------------------------------------------ host.imread
def _pil_bgr(path):
    from PIL import Image, ImageOps
    with Image.open(path) as im:
        return np.asarray(ImageOps.exif_transpose(im).convert("RGB"))[:, :, ::-1]


@pytest.mark.parametrize("ext,mode", [("png", "RGB"), ("png", "L"), ("png", "P"), ("png", "RGBA"), ("jpg", "RGB"),
                                      ("jpg", "L")])
def test_imread_modes(tmp_path, ext, mode):
    from PIL import Image
    rng = np.random.RandomState(3)
    rgb = rng.randint(0, 256, (37, 53, 3)).astype(np.uint8)
    im = Image.fromarray(rgb)
    if mode == "L":
        im = im.convert("L")
    elif mode == "P":
        im = im.quantize(64)
    elif mode == "RGBA":
        im = Image.fromarray(np.concatenate([rgb, rng.randint(0, 256, (37, 53, 1)).astype(np.uint8)], 2), "RGBA")
    path = str(tmp_path / ("x." + ext))
    im.save(path)
    got = host.imread(path)
    assert got.dtype == np.uint8 and got.shape == (37, 53, 3) and got.flags.c_contiguous
    assert np.array_equal(got, _pil_bgr(path))
    if mode == "RGB" and ext == "png":
        assert np.array_equal(got, rgb[:, :, ::-1])          # BGR: channel 0 is blue
    if mode == "L":
        assert np.array_equal(got[:, :, 0], got[:, :, 1]) and np.array_equal(got[:, :, 1], got[:, :, 2])
    if mode == "RGBA" and ext == "png":
        assert np.array_equal(got, rgb[:, :, ::-1])          # alpha dropped, colour untouched


@pytest.mark.parametrize("orientation,rotate", [(3, 2), (6, -1), (8, 1)])
def test_imread_applies_exif_orientation(tmp_path, orientation, rotate):
    """Orientation 3 is a half turn, 6 a quarter turn clockwise, 8 counter-clockwise (applied as IMREAD_COLOR does)."""
    from PIL import Image
    rgb = np.zeros((20, 40, 3), np.uint8)
    rgb[:, :20] = (255, 0, 0)
    rgb[:, 20:] = (0, 0, 255)
    exif = Image.Exif()
    exif[0x0112] = orientation
    path = str(tmp_path / "o.png")
    Image.fromarray(rgb).save(path, exif=exif)
    got = host.imread(path)
    assert np.array_equal(got, np.ascontiguousarray(np.rot90(rgb, rotate)[:, :, ::-1]))
    jpath = str(tmp_path / "o.jpg")
    Image.fromarray(rgb).save(jpath, exif=exif, quality=100)
    j = host.imread(jpath)
    assert j.shape == got.shape and np.array_equal(j, _pil_bgr(jpath))


def test_imread_names_the_missing_or_broken_file(tmp_path):
    missing = str(tmp_path / "nope.jpg")
    with pytest.raises(OSError, match="nope.jpg"):
        host.imread(missing)
    broken = tmp_path / "broken.jpg"
    broken.write_bytes(b"not an image")
    with pytest.raises(OSError, match="broken.jpg"):
        host.imread(str(broken))


# ------------------------------------------------------------------------------------------------ datasets on disk
def _mirrored(a, b):
    """b is a's flipped entry: boxes mirrored in the width, the rest shared."""
    x = b["boxes"]
    return (np.array_equal(x[:, 0], a["width"] - a["boxes"][:, 2] - 1)
            and np.array_equal(x[:, 2], a["width"] - a["boxes"][:, 0] - 1)
            and np.array_equal(x[:, 1::2], a["boxes"][:, 1::2]) and b["flipped"] and not a["flipped"]
            and b["image"] == a["image"] and b["max_overlaps"] is a["max_overlaps"])


def test_voc_devkit_flip_merge_filter(tmp_path):
    dk, listing = TD.write_voc(str(tmp_path))
    cfg = IT.default_config(dataset="pascal_voc")
    assert cfg.TRAIN.FLIP and cfg.dataset.dataset == "PascalVOC"
    roidbs = []
    for s in ("2007_trainval", "2012_trainval"):
        r = load_data.load_proposal_roidb(cfg.dataset.dataset, s, str(tmp_path), dk, flip=cfg.TRAIN.FLIP, only_gt=True,
                                          device="cpu")
        n = len(listing[s])
        assert len(r) == 2 * n
        assert all(_mirrored(a, b) for a, b in zip(r[:n], r[n:]))
        assert all(e["boxes"].dtype == np.float32 for e in r)
        roidbs.append(r)
    names = [os.path.basename(e["image"])[:-4] for e in roidbs[0] + roidbs[1]]
    merged = load_data.merge_roidb(roidbs)
    assert [os.path.basename(e["image"])[:-4] for e in merged] == names
    want = [n for s in ("2007_trainval", "2012_trainval") for n, _, _, _ in listing[s] * 2]
    assert names == want                                               # 2007 (and its flips), then 2012
    kept = load_data.filter_roidb(list(merged), cfg)
    usable = [e for e in merged if len(e["boxes"]) > 0]                 # only GT rows: usable = non-difficult objects
    assert [id(e) for e in kept] == [id(e) for e in usable] and len(kept) == len(merged) - 4
    means, stds = load_data.add_bbox_regression_targets(kept, cfg)
    assert np.array_equal(means, np.tile([0.0, 0.0, 0.0, 0.0], 2)) and np.array_equal(stds, np.tile([0.1, 0.1, 0.2, 0.2], 2))
    for e in kept:                                                      # every GT row regresses to itself
        assert e["bbox_targets"].shape == (len(e["boxes"]), 5)
        assert np.array_equal(e["bbox_targets"][:, 0], e["max_classes"])
        assert np.abs(e["bbox_targets"][:, 1:]).max() < 1e-6     # log(w / (w + 1e-7))


def test_coco_image_set_and_scales(tmp_path):
    dp = TD.write_coco(str(tmp_path))
    cfg = IT.default_config(neg=False)
    assert cfg.dataset.dataset == "coco" and cfg.dataset.NUM_CLASSES == 81
    assert load_data.paper_train_scales(cfg) == (3.0, 1.667, 512.0) and cfg.TRAIN.SCALES == (3.0, 1.667, 512.0)
    voc = IT.default_config(dataset="pascal_voc")
    scales = list(voc.TRAIN.SCALES)
    assert load_data.paper_train_scales(voc) == scales
    r = load_data.load_proposal_roidb("coco", "train2014", str(tmp_path), dp, flip=True, only_gt=True, device="cpu")
    assert len(r) == 6 and all(_mirrored(a, b) for a, b in zip(r[:3], r[3:]))
    kept = load_data.filter_roidb(r, cfg)
    assert len(kept) == 4 and all(len(e["boxes"]) for e in kept)
    with pytest.raises(ValueError, match="dataset must be one of"):
        load_data.load_proposal_roidb("pascal_voc", "2007_trainval", str(tmp_path), dp)


def test_image_data_is_shared_with_the_flipped_entry():
    im = np.zeros((4, 6, 3), np.uint8)
    roidb = [dict(image="a.jpg", image_data=im, width=6, height=4, boxes=np.array([[0, 1, 2, 3]], np.float32),
                  gt_classes=np.ones(1, np.int32), gt_overlaps=np.zeros((1, 2), np.float32),
                  max_classes=np.ones(1), max_overlaps=np.ones(1, np.float32), flipped=False)]
    imdb = types.SimpleNamespace(image_set_index=["a"])
    out = load_data.append_flipped_images(imdb, roidb)
    assert out[1]["image_data"] is im and out[1]["boxes"].tolist() == [[3, 1, 5, 3]] and imdb.image_set_index == ["a", "a"]


def _first_batch(entry, cfg):
    np.random.seed(4)
    host.srand(4)
    it = IT.MNIteratorE2E([entry], cfg, batch_size=1, image_loader=host.imread, n_buffers=3)
    raw = it._get_batch()
    h, w = int(raw.table[0, 1]), int(raw.table[0, 2])
    pix = raw.pixels.numpy()[:h * w * 3].reshape(h, w, 3).copy()
    return it.roidb[0]["crops"], pix, raw.table[0].clone(), raw.gt_boxes[0].clone()


def test_iterator_chips_of_a_flipped_entry_are_mirror_images(tmp_path):
    """A flipped entry read from its JPEG (host.imread) and the same entry with its pixels mirrored in memory and
    flipped=False: the same chips and GT, and the source rectangle of the flipped one is the other's mirrored (the
    device flips it back, sniper_chip_input)."""
    dk, _ = TD.write_voc(str(tmp_path), sets=(("2007", "trainval", 2),), size=(400, 300), empty_last=False)
    cfg = IT.default_config(neg=False, dataset="pascal_voc")
    r = load_data.load_proposal_roidb("PascalVOC", "2007_trainval", str(tmp_path), dk, flip=True, only_gt=True,
                                      device="cpu")
    for e in r[2:]:
        twin = dict(e, flipped=False, image_data=np.ascontiguousarray(host.imread(e["image"])[:, ::-1]))
        crops_f, pix_f, tab_f, gt_f = _first_batch(dict(e), cfg)
        crops_t, pix_t, tab_t, gt_t = _first_batch(twin, cfg)
        assert len(crops_f) > 0 and np.array_equal([c[0] for c in crops_f], [c[0] for c in crops_t])
        assert int(tab_f[5]) == 1 and int(tab_t[5]) == 0 and np.array_equal(tab_f[1:5], tab_t[1:5])
        assert np.array_equal(pix_f[:, ::-1], pix_t) and np.array_equal(gt_f, gt_t)
