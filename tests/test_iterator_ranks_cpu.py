"""Data-parallel training iterator on the host: `MNIteratorE2E(batch_size=W*B, nGPUs=W, rank=r, seed=s)` yields, batch
for batch, chips [r*B, (r+1)*B) of the global batch the rank=None iterator with the same seed yields -- pixels, chip
table, ranges, GT bookkeeping, FocusPixel boxes, subsampling seed -- over flipped entries, negative chips, AutoFocus, a
VOCdevkit read from disk and epochs that need padding.  The seed=None path is pinned to the bytes the iterator produced
before ranks existed, and the plan check of Trainer.fit is run on a gloo world of two."""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from sniper_b200 import _lib, host, load_data  # noqa: E402
from sniper_b200 import iterator as IT  # noqa: E402


def _snap(raw):
    """A copy of one raw batch (the iterator refills its buffers), each chip's pixels cut out by its table row."""
    t = raw.table.numpy().copy()
    pix = raw.pixels.numpy()
    B = t.shape[0]
    ngt, ninv = raw.ngt.numpy().copy(), raw.ninv.numpy().copy()
    s = dict(table=t, seed=raw.seed, chip_base=raw.chip_base, digest=raw.plan_digest, used=raw.used_pixels,
             pixels=[pix[o:o + h * w * 3].tobytes() for o, h, w in t[:, :3]],
             valid_ranges=raw.valid_ranges.numpy().copy(), im_info=raw.im_info.numpy().copy(),
             anchor_im_info=raw.anchor_im_info.numpy().copy(), ngt=ngt, ninv=ninv,
             gt_valid=[raw.gt_valid[k, :ngt[k]].numpy().copy() for k in range(B)],
             gt_invalid=[raw.gt_invalid[k, :ninv[k]].numpy().copy() for k in range(B)],
             gt_boxes=raw.gt_boxes.numpy().copy())
    if raw.focus_boxes is not None:
        nf = raw.nfocus.numpy().copy()
        s.update(nfocus=nf, focus_boxes=[raw.focus_boxes[k, :nf[k]].numpy().copy() for k in range(B)])
    return s


def _epochs(it, n=2):
    """[(len(it), [raw batch copies])] of n epochs."""
    out = []
    for e in range(n):
        if e:
            it.reset()
        out.append((len(it), [_snap(raw) for raw in it]))
    return out


def _copy(roidb):
    """The iterator keeps its per-epoch state in the roidb entries; each rank has its own roidb."""
    return [dict(r) for r in roidb]


def _check_slices(roidb, cfg, W, B, seed, loader=None):
    full_it = IT.MNIteratorE2E(_copy(roidb), cfg, batch_size=W * B, nGPUs=W, seed=seed, image_loader=loader)
    full = _epochs(full_it)
    assert all(g["chip_base"] == 0 for _, ep in full for g in ep)
    for r in range(W):
        it = IT.MNIteratorE2E(_copy(roidb), cfg, batch_size=W * B, nGPUs=W, rank=r, seed=seed, image_loader=loader)
        mine = _epochs(it)
        for (n_full, ep_full), (n_mine, ep_mine) in zip(full, mine):
            # the global, padded chip count on every rank, and the same number of batches
            assert n_mine == n_full == len(ep_full) * W * B and len(ep_mine) == len(ep_full) > 0
            for g, m in zip(ep_full, ep_mine):
                base = r * B
                sl = slice(base, base + B)
                assert m["chip_base"] == base and m["seed"] == g["seed"] and m["digest"] == g["digest"]
                assert m["pixels"] == g["pixels"][sl]
                assert np.array_equal(m["table"][:, 1:], g["table"][sl, 1:])
                assert m["table"][0, 0] == 0 and m["used"] == sum(len(p) for p in m["pixels"])
                for k in ("valid_ranges", "im_info", "anchor_im_info", "ngt", "ninv", "gt_boxes"):
                    assert m[k].tobytes() == g[k][sl].tobytes(), k
                for k in ("gt_valid", "gt_invalid") + (("focus_boxes",) if "nfocus" in g else ()):
                    assert all(a.tobytes() == b.tobytes() for a, b in zip(m[k], g[k][sl])), k
                if "nfocus" in g:
                    assert m["nfocus"].tobytes() == g["nfocus"][sl].tobytes()
    padded = full_it.chip_count % (W * B) != 0
    return full, padded


@pytest.mark.parametrize("case", ["neg_flipped", "autofocus"])
def test_rank_slices_equal_the_global_batch_synthetic(case):
    cfg = IT.default_config(neg=True, autofocus=case == "autofocus")
    roidb = IT.synthetic_roidb(4, seed=3, n_prop=300)
    assert any(r["flipped"] for r in roidb) and not all(r["flipped"] for r in roidb)
    padded = []
    for W in (2, 3):
        for B in (1, 2):
            full, p = _check_slices(roidb, cfg, W, B, seed=11)
            padded.append(p)
            if case == "neg_flipped" and W == 2 and B == 1:
                it = IT.MNIteratorE2E(_copy(roidb), cfg, batch_size=2, nGPUs=2, rank=0, seed=11)
                assert any(len(r["neg_crops"]) > 0 for r in it.roidb)         # negative chips were drawn
            if case == "autofocus":
                assert any(int(g["nfocus"].sum()) > 0 for _, ep in full for g in ep)
    assert any(padded)         # at least one (W, B) whose chip count is not a multiple of the global batch


def test_rank_slices_equal_the_global_batch_voc_from_disk(tmp_path):
    import train_data_fixture as TD
    dk, _ = TD.write_voc(str(tmp_path), sets=(("2007", "trainval", 4),), empty_last=False)
    cfg = IT.default_config(neg=False, dataset="pascal_voc")
    roidb = load_data.load_proposal_roidb("PascalVOC", "2007_trainval", str(tmp_path), dk, flip=True, only_gt=True,
                                          device="cpu")
    assert any(r["flipped"] for r in roidb)
    for W in (2, 3):
        for B in (1, 2):
            _check_slices(roidb, cfg, W, B, seed=4, loader=host.imread)


def test_epoch_plans_are_a_function_of_the_seed():
    cfg = IT.default_config(neg=True)
    roidb = IT.synthetic_roidb(4, seed=3, n_prop=300)
    d = []
    for seed in (5, 5, 6):
        np.random.seed(len(d))             # the global state must not matter
        host.srand(len(d))
        it = IT.MNIteratorE2E(_copy(roidb), cfg, batch_size=4, nGPUs=2, rank=1, seed=seed)
        first = it.plan_digest
        it.reset()
        d.append((first, it.plan_digest, it.inds.tobytes()))
    assert d[0] == d[1] and d[0][0] != d[2][0] and d[0][0] != d[0][1]


def test_rank_needs_a_seed_and_a_valid_rank():
    cfg = IT.default_config(neg=False)
    roidb = IT.synthetic_roidb(1, seed=1, n_prop=10)
    with pytest.raises(ValueError, match="needs a seed"):
        IT.MNIteratorE2E(roidb, cfg, batch_size=4, nGPUs=2, rank=0)
    with pytest.raises(ValueError, match="not in"):
        IT.MNIteratorE2E(roidb, cfg, batch_size=4, nGPUs=2, rank=2, seed=0)
    assert _lib.SIGNATURES["sniper_anchor_subsample_at"] == ("i", "pppiiiiiiuip")


# sha256 of every raw batch of two epochs per configuration, written by the iterator before it had `rank` / `seed`
# (np.random.seed(k) and host.srand(k) first): the seed=None path must keep producing these bytes
_UNSEEDED_SHA256 = {
    "neg": "e95ac9e45f9531ac7f8869f8b3f6e30a1ee749dbefebb09536a48bda4229ffb5",
    "autofocus": "d1a743f84cbbaa2afdfe19df2c6e582bdd1e4e3e0b356d931eb6ce902b2bcebf",
}


def _unseeded_sha256(case):
    cfg = IT.default_config(neg=True, autofocus=case == "autofocus")
    roidb = IT.synthetic_roidb(5, seed=2, n_prop=300)
    np.random.seed(9)
    host.srand(9)
    it = IT.MNIteratorE2E(roidb, cfg, batch_size=3)
    h = hashlib.sha256()
    for e in range(2):
        if e:
            it.reset()
        for raw in it:
            B = raw.table.shape[0]
            ngt, ninv = raw.ngt.numpy(), raw.ninv.numpy()
            parts = [raw.pixels.numpy()[:raw.used_pixels], raw.table.numpy(), raw.valid_ranges.numpy(),
                     raw.im_info.numpy(), raw.anchor_im_info.numpy(), ngt, ninv, raw.gt_boxes.numpy(),
                     np.int64(raw.seed)]
            parts += [raw.gt_valid[k, :ngt[k]].numpy() for k in range(B)]
            parts += [raw.gt_invalid[k, :ninv[k]].numpy() for k in range(B)]
            if raw.focus_boxes is not None:
                nf = raw.nfocus.numpy()
                parts += [nf] + [raw.focus_boxes[k, :nf[k]].numpy() for k in range(B)]
            for p in parts:
                h.update(np.ascontiguousarray(p).tobytes())
    return h.hexdigest()


@pytest.mark.parametrize("case", ["neg", "autofocus"])
def test_unseeded_iterator_keeps_its_bytes(case):
    assert _unseeded_sha256(case) == _UNSEEDED_SHA256[case]


# ---------------------------------------------------------------- the plan check of Trainer.fit, two gloo ranks
def _plan_rank(rank, port, seeds, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=2)
    sys.path.insert(0, ROOT)
    from sniper_b200 import iterator, trainer
    cfg = iterator.default_config(neg=True)
    roidb = iterator.synthetic_roidb(3, seed=3, n_prop=300)
    it = iterator.MNIteratorE2E(roidb, cfg, batch_size=4, nGPUs=2, rank=rank, seed=seeds[rank])
    try:
        trainer.check_plan(next(it).plan_digest, 2, epoch=0)
        q.put((rank, "ok"))
    except ValueError as e:
        q.put((rank, str(e)))
    dist.destroy_process_group()


@pytest.mark.parametrize("seeds", [(7, 7), (7, 8)], ids=["same", "different"])
def test_plan_check_gloo_world2(seeds):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29661 + (seeds[0] != seeds[1])
    procs = [ctx.Process(target=_plan_rank, args=(r, port, seeds, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = sorted(q.get(timeout=180) for _ in procs)
    finally:
        for p in procs:
            p.join(60)
            if p.is_alive():
                p.kill()
    assert [r for r, _ in res] == [0, 1]
    if seeds[0] == seeds[1]:
        assert all(m == "ok" for _, m in res), res
    else:
        for _, m in res:
            assert m.startswith("epoch 0: the ranks' epoch plans differ") and "ranks [0]" in m and "ranks [1]" in m, m
