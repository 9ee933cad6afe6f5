"""The device input stage of a data-parallel rank: `sniper_anchor_subsample_at` keys its draws by the chip's position in
the global batch, so each rank's InputStage outputs are byte-equal to the matching rows of the global batch's."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sniper_b200 import iterator as IT  # noqa: E402
from sniper_b200._lib import check, lib  # noqa: E402

pytestmark = pytest.mark.gpu


def _labels(B, A, H, W, seed):
    """Random labels with more positives / negatives than the subsampling keeps, and matching regression weights."""
    rng = np.random.RandomState(seed)
    n = A * H * W
    lab = np.full((B, n), -1, np.float32)
    for b in range(B):
        idx = rng.permutation(n)
        nfg = int(rng.randint(100, 400))
        lab[b, idx[:nfg]] = 1
        lab[b, idx[nfg:nfg + int(rng.randint(500, 5000))]] = 0
    bw = np.zeros((B, 4 * A, H * W), np.float32)
    for b in range(B):
        fg = np.where(lab[b] == 1)[0]
        for j in range(4):
            bw[b, 4 * (fg // (H * W)) + j, fg % (H * W)] = 1
    bt = rng.randn(B, 4 * A, H * W).astype(np.float32) * bw
    return lab, bt, bw


def _subsample(lab, bt, bw, A, H, W, seed, chip_base=None):
    t = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (lab, bt, bw)]
    st = torch.cuda.current_stream().cuda_stream
    ptr = [x.data_ptr() for x in t]
    if chip_base is None:
        check(lib().sniper_anchor_subsample(*ptr, lab.shape[0], A, H, W, 128, 256, seed, st))
    else:
        check(lib().sniper_anchor_subsample_at(*ptr, lab.shape[0], A, H, W, 128, 256, seed, chip_base, st))
    return [x.cpu().numpy() for x in t]


def test_subsample_at_keys_by_global_chip():
    A, H, W = 21, 32, 32
    lab, bt, bw = _labels(7, A, H, W, seed=3)
    plain = _subsample(lab, bt, bw, A, H, W, 1234)
    at0 = _subsample(lab, bt, bw, A, H, W, 1234, chip_base=0)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(plain, at0))
    assert (plain[0] != lab).any()                          # the subsampling dropped anchors
    for k, n in ((1, 3), (4, 2), (6, 1)):
        # chips [k, k + n) of the wide launch, launched alone: chip_base = k draws what the wide launch drew for them
        part = _subsample(lab[k:k + n], bt[k:k + n], bw[k:k + n], A, H, W, 1234, chip_base=k)
        assert all(p.tobytes() == w[k:k + n].tobytes() for p, w in zip(part, plain)), (k, n)
        other = _subsample(lab[k:k + n], bt[k:k + n], bw[k:k + n], A, H, W, 1234, chip_base=k + 1)
        assert other[0].tobytes() != plain[0][k:k + n].tobytes()


@pytest.mark.parametrize("autofocus", [False, True], ids=["plain", "autofocus"])
def test_rank_input_stage_rows_equal_the_global_batch(autofocus):
    W, B, seed = 2, 2, 21
    cfg = IT.default_config(neg=True, autofocus=autofocus)
    roidb = IT.synthetic_roidb(4, seed=5, n_prop=300)
    full_it = IT.MNIteratorE2E([dict(r) for r in roidb], cfg, batch_size=W * B, nGPUs=W, seed=seed)
    rank_its = [IT.MNIteratorE2E([dict(r) for r in roidb], cfg, batch_size=W * B, nGPUs=W, rank=r, seed=seed)
                for r in range(W)]
    full_stage = IT.InputStage(cfg, "cuda", W * B)
    rank_stages = [IT.InputStage(cfg, "cuda", B) for _ in range(W)]
    keys = ["data", "label", "bbox_target", "bbox_weight", "gt_boxes", "valid_ranges", "im_info"]
    if autofocus:
        keys.append("scale_label")
    dropped = 0
    n = 0
    for raws in zip(full_it, *rank_its):
        full = {k: v.clone() for k, v in full_stage.run(raws[0]).items()}
        before = full_stage.run(raws[0], subsample=False)["label"]
        dropped += int((before != full["label"]).sum())
        for r in range(W):
            out = rank_stages[r].run(raws[1 + r])
            for k in keys:
                assert out[k].shape[0] == B
                assert out[k].cpu().numpy().tobytes() == full[k][r * B:(r + 1) * B].cpu().numpy().tobytes(), (n, r, k)
        n += 1
    assert n == len(full_it) // (W * B) and n > 0
    assert dropped > 0                     # the subsampling dropped anchors, per global chip position
