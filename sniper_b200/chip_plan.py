"""The training epoch plan on the device: what `chip_worker.chip_extractor` and `chip_worker.box_assigner` compute for
every roidb entry (positive chips per scale, box -> chip assignment, negative chips), with the same types, values and
order, in a few launches per epoch instead of two Python loops over the roidb.

One (entry, scale) problem of the host is a "call": one greedy cover (`host.chips_generate`) and one `_assign`.  The
host path's draws from the C `rand()` stream are part of the plan: each cover with boxes shuffles its candidates with
n_cand - 1 draws, every entry's positive covers first (entry-major, scale-minor), then every entry's negative covers.
Which covers draw depends only on the geometry and on which covers have boxes, so an epoch runs in two phases:

1. positives: `sniper_chip_plan_count` gives each call's GT box count, the host draws the candidate orders of the calls
   with boxes (`sniper_chips_shuffle`), then `sniper_chip_plan_cover` and `sniper_chip_plan_assign` (mode 0) give the
   chips and every box's owner, and so the boxes no positive chip kept;
2. negatives: the host draws the orders of the calls with uncovered boxes, then the cover and the assignment run again
   in mode 1.

The roidb is cut into chunks of entries, so the candidate orders and the per-chunk outputs stay bounded; rand() is drawn
chunk by chunk in the host's order.  The boxes, their integer sizes (`_int_sizes`, in the roidb's own dtype) and the GT
flags are computed once and kept on the device, up to `resident_bytes`; chunks past that are uploaded when they are
planned.  The geometry (`image_scales`, the scaled image sizes) and the roidb's boxes are read once, at construction:
an entry changed afterwards is not seen.  The `/ f` of the chips and the chip tags stay in numpy, as the host has them."""
import numpy as np
import torch

from . import _lib as _libmod
from ._lib import check, lib
from .chip_worker import image_scales

TABLE_COLS = 16
(C_ENTRY, C_SCALE, C_KIND, C_W, C_H, C_NCAND, C_NBOX, C_PERM, C_OUT, C_CAP, C_WS, C_F, C_THR, C_LO, C_HI,
 C_F32) = range(TABLE_COLS)
HOST_CAP = 4096         # host.chips_generate keeps the first 4096 chips of a cover


def n_candidates(W, H, chip_size, stride):
    """The candidate count of sniper_chips_generate for scaled image sizes W, H (integer arrays)."""
    W, H = np.asarray(W, np.int64), np.asarray(H, np.int64)
    nx = np.where(W > chip_size, (W - chip_size + stride - 1) // stride, 0)
    ny = np.where(H > chip_size, (H - chip_size + stride - 1) // stride, 0)
    return 3 + nx * ny + ny + nx


def chips_shuffle(n_cand):
    """The candidate orders a sequence of host.chips_generate calls with n_cand[c] candidates draws from rand() (0: a
    call without boxes, no draw), back to back as int32; rand() ends where those calls leave it."""
    n_cand = np.ascontiguousarray(n_cand, np.int32).reshape(-1)
    perm = np.empty(max(int(n_cand.astype(np.int64).sum()), 1), np.int32)
    check(lib().sniper_chips_shuffle(n_cand.ctypes.data, len(n_cand), perm.ctypes.data))
    return perm


def _ranges(starts, lens):
    """concatenate(arange(s, s + n) for s, n in zip(starts, lens))"""
    lens = np.asarray(lens, np.int64)
    total = int(lens.sum())
    if total == 0:
        return np.zeros(0, np.int64)
    first = np.cumsum(lens) - lens
    return np.repeat(np.asarray(starts, np.int64) - first, lens) + np.arange(total)


def _box_arrays(boxes_list, int_sizes):
    """float32 boxes, int32 [n, 2] (w, h) and the float32-scaling flag of every entry.  w, h come from
    chip_worker._int_sizes in each entry's own dtype (uint16 subtraction wraps as the host's does)."""
    n = np.array([len(b) for b in boxes_list], np.int64)
    off = np.zeros(len(n) + 1, np.int64)
    np.cumsum(n, out=off[1:])
    boxes = np.zeros((int(off[-1]), 4), np.float32)
    wh = np.zeros((int(off[-1]), 2), np.int32)
    f32 = np.zeros(len(n), np.int64)
    by_dtype = {}
    for e, b in enumerate(boxes_list):
        by_dtype.setdefault(np.asarray(b).dtype, []).append(e)
    for dt, es in by_dtype.items():
        if dt == np.float16 or dt.kind not in "fiu":
            raise ValueError("device chip plan: roidb boxes of dtype %s are not supported" % dt)
        b = np.concatenate([np.asarray(boxes_list[e]).reshape(-1, 4) for e in es])
        b32 = b.astype(np.float32)
        if dt != np.float32 and not np.array_equal(b32.astype(np.float64), b.astype(np.float64)):
            raise ValueError("device chip plan: %s roidb boxes must be exact in float32" % dt)
        w, h, _, _ = int_sizes(b)
        rows = _ranges(off[es], n[es])
        boxes[rows], wh[rows, 0], wh[rows, 1] = b32, w, h
        f32[es] = dt == np.float32
    return off, boxes, wh, f32


class DevicePlan(object):
    """chip_worker's epoch plan for a fixed roidb on one device.  `plan(roidb)` fills r['crops'] and
    r['props_in_chips'] of every entry, and with TRAIN.USE_NEG_CHIPS r['neg_chips'] / r['neg_crops'] (the same list)
    and r['neg_props_in_chips'], as chip_extractor + box_assigner with the worker's current chip stride would, drawing
    the same values from rand().  It runs on its own CUDA stream and synchronises only that stream."""

    def __init__(self, roidb, worker, device=None, chunk_images=8192, resident_bytes=4 << 30):
        self.worker = worker
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.type != "cuda":
            raise ValueError("DevicePlan: device must be a CUDA device, not %s" % self.device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.stream = torch.cuda.Stream(device=self.device)
        S = len(worker.scales)
        self.S, self.n = S, len(roidb)
        self.use_neg = bool(worker.use_neg_chips)
        # per (entry, scale): the factor, the scaled image size and the chip tags (stride-independent)
        f = np.zeros((self.n, S))
        for e, r in enumerate(roidb):
            f[e] = image_scales(worker.scales, r['width'], r['height'])
        self.f = f
        self.W = np.array([[int(r['width'] * x) for x in fe] for r, fe in zip(roidb, f)], np.int64).reshape(self.n, S)
        self.H = np.array([[int(r['height'] * x) for x in fe] for r, fe in zip(roidb, f)], np.int64).reshape(self.n, S)
        self.tags = [[worker._tag(None, float(f[e, s]), s, r)[1:] for s in range(S)] for e, r in enumerate(roidb)]
        self.box_off, self.boxes, self.wh, self.f32 = _box_arrays([r['boxes'] for r in roidb], worker._int_sizes)
        self.gt = np.concatenate([np.asarray(r['max_overlaps']).reshape(-1) == 1 for r in roidb] +
                                 [np.zeros(0, bool)]).astype(np.uint8)
        if len(self.gt) != len(self.boxes):
            raise ValueError("device chip plan: every entry needs one max_overlaps value per box")
        kind = np.where(np.arange(S) == S - 1, 2, np.where(np.arange(S) == 0, 0, 1))
        vr = np.array([[float(v[0]), float(v[1])] for v in worker.valid_ranges[:S]], np.float64).reshape(S, 2)
        self.kind, self.lo, self.hi = kind, vr[:, 0].copy(), vr[:, 1].copy()
        self.chunks = [(e0, min(e0 + chunk_images, self.n)) for e0 in range(0, self.n, max(int(chunk_images), 1))]
        self.resident_bytes = int(resident_bytes)
        self._resident = {}
        self.stats = {}

    # ---------------------------------------------------------------- device data of a chunk
    def _static(self, ci):
        d = self._resident.get(ci)
        if d is not None:
            return d
        e0, e1 = self.chunks[ci]
        b0, b1 = int(self.box_off[e0]), int(self.box_off[e1])
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.device)  # noqa: E731
        d = dict(box_off=up(self.box_off[e0:e1 + 1] - b0), boxes=up(self.boxes[b0:b1].reshape(-1, 4)),
                 wh=up(self.wh[b0:b1].reshape(-1, 2)), gt=up(self.gt[b0:b1]), nbox=b1 - b0)
        nbytes = sum(t.numel() * t.element_size() for t in d.values() if torch.is_tensor(t))
        self.stats["h2d_bytes"] += nbytes
        held = sum(x["bytes"] for x in self._resident.values())
        if held + nbytes <= self.resident_bytes:
            d["bytes"] = nbytes
            self._resident[ci] = d
        return d

    def resident_device_bytes(self):
        """Device bytes the plan keeps between epochs (the resident chunks' boxes, sizes and GT flags)."""
        return sum(x["bytes"] for x in self._resident.values())

    def _table(self, ci, n_cand, thr):
        e0, e1 = self.chunks[ci]
        ne, S = e1 - e0, self.S
        t = np.zeros((ne * S, TABLE_COLS), np.int64)
        t[:, C_ENTRY] = np.repeat(np.arange(ne), S)
        t[:, C_SCALE] = np.tile(np.arange(S), ne)
        t[:, C_KIND] = np.tile(self.kind, ne)
        t[:, C_W], t[:, C_H] = self.W[e0:e1].reshape(-1), self.H[e0:e1].reshape(-1)
        t[:, C_NCAND] = n_cand[e0:e1].reshape(-1)
        t[:, C_F] = np.ascontiguousarray(self.f[e0:e1]).reshape(-1).view(np.int64)
        t[:, C_THR] = np.ascontiguousarray(thr[e0:e1]).reshape(-1).view(np.int64)
        t[:, C_LO] = np.tile(self.lo, ne).view(np.int64)
        t[:, C_HI] = np.tile(self.hi, ne).view(np.int64)
        t[:, C_F32] = np.repeat(self.f32[e0:e1], S)
        return t

    def _cover_assign(self, t, d, nbox, mode, pos_owner):
        """Draws the calls' candidate orders, runs the cover and the assignment of one chunk; returns the chips
        (float32, host), their per-call count and slot offset, the owners (device and host) and the per-call count of
        selected boxes no chip kept."""
        L = lib()
        cs, stride = int(self.worker.chip_size), int(self.worker.chip_stride)
        n_cand = t[:, C_NCAND]
        draw = np.where(nbox > 0, n_cand, 0)
        perm = chips_shuffle(draw)
        t[:, C_NBOX] = nbox
        t[:, C_PERM] = np.cumsum(draw) - draw
        cap = np.where(nbox > 0, np.minimum(n_cand, nbox), 0)
        t[:, C_OUT] = np.cumsum(cap) - cap
        t[:, C_CAP] = cap
        ws_bytes = np.zeros(1, np.int64)
        check(L.sniper_chip_plan_layout(t.ctypes.data, len(t), cs, stride, ws_bytes.ctypes.data))
        dev = self.device
        n_calls, total = len(t), max(int(cap.sum()), 1)
        d_t = torch.from_numpy(t).to(dev)
        d_perm = torch.from_numpy(perm).to(dev)
        ws = torch.empty(int(ws_bytes[0]), dtype=torch.uint8, device=dev) if ws_bytes[0] else None
        chips32 = torch.empty((total, 4), dtype=torch.float32, device=dev)
        chips64 = torch.empty((total, 4), dtype=torch.float64, device=dev)
        nchips = torch.empty(max(n_calls, 1), dtype=torch.int32, device=dev)
        owner = torch.empty((max(d["nbox"], 1), self.S), dtype=torch.int16, device=dev)
        left = torch.empty(max(n_calls, 1), dtype=torch.int32, device=dev)
        st = self.stream.cuda_stream
        p = lambda x: 0 if x is None else x.data_ptr()  # noqa: E731
        ev = self._events()
        check(L.sniper_chip_plan_cover(p(d_t), t.ctypes.data, n_calls, mode, self.S, cs, stride, p(d["box_off"]),
                                       p(d["boxes"]), p(d["wh"]), p(d["gt"]), p(pos_owner), p(d_perm), p(ws),
                                       int(ws_bytes[0]), p(chips32), p(chips64), p(nchips), st))
        check(L.sniper_chip_plan_assign(p(d_t), t.ctypes.data, n_calls, mode, self.S, p(d["box_off"]), p(d["boxes"]),
                                        p(d["wh"]), p(pos_owner), p(chips64), p(nchips), p(owner), p(left), st))
        ev[1].record(self.stream)
        self.stats["h2d_bytes"] += t.nbytes + perm.nbytes
        self.stats["launches"] += 2
        nch = nchips.cpu().numpy()[:n_calls].astype(np.int64)
        self.stats["kernel_ms"] += ev[0].elapsed_time(ev[1])
        if (nch < 0).any():
            c = int(np.flatnonzero(nch < 0)[0])
            raise _libmod.SniperError("device chip plan: call %d: the table disagrees with the boxes it selects" % c)
        out = dict(chips=chips32.cpu().numpy(), nch=np.minimum(nch, HOST_CAP), off=t[:, C_OUT].copy(),
                   owner_dev=owner, owner=owner.cpu().numpy()[:d["nbox"]], left=left.cpu().numpy()[:n_calls])
        self.stats["d2h_bytes"] += chips32.numel() * 4 + owner.numel() * 2 + 2 * n_calls * 4
        return out

    def _events(self):
        """A start event recorded on the plan stream now and an end event for the caller: stats['kernel_ms'] sums the
        time between them."""
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record(self.stream)
        return ev

    # ---------------------------------------------------------------- host-side lists
    def _chips(self, ci, res):
        """Per entry of the chunk: the chips (float64 rows = float32 chip / f) in (scale, pick) order, their scale
        index, and the first chip of each (entry, scale)."""
        e0, e1 = self.chunks[ci]
        ne, S = e1 - e0, self.S
        nch = res["nch"]
        idx = _ranges(res["off"], nch)
        xyxy = res["chips"][idx].astype(np.float64) / np.repeat(self.f[e0:e1].reshape(-1), nch)[:, None]
        first = np.zeros(ne * S + 1, np.int64)
        np.cumsum(nch, out=first[1:])
        return xyxy, np.repeat(np.tile(np.arange(S), ne), nch), first

    def _lists(self, ci, owner, first, n_chips):
        """The box ids of every chip (chunk-wide chip index), in box order: boxes (b, s) with owner o >= 0 belong to
        chip first[entry(b) * S + s] + o."""
        e0, e1 = self.chunks[ci]
        b0 = int(self.box_off[e0])
        nb = np.diff(self.box_off[e0:e1 + 1])
        entry = np.repeat(np.arange(e1 - e0), nb)
        b, s = np.nonzero(owner >= 0)
        chip = first[entry[b] * self.S + s] + owner[b, s]
        order = np.argsort(chip, kind="stable")
        local = (b - (self.box_off[e0 + entry[b]] - b0))[order]
        cnt = np.bincount(chip, minlength=n_chips)
        return local, cnt

    def plan(self, roidb):
        """Fills the roidb's plan for the worker's current chip stride (see the class).  self.stats then holds the
        epoch's H2D / D2H bytes, launches and the CUDA-event time of the launches (kernel_ms)."""
        if len(roidb) != self.n:
            raise ValueError("DevicePlan: built for %d entries, given %d" % (self.n, len(roidb)))
        w = self.worker
        S, cs, stride = self.S, int(w.chip_size), int(w.chip_stride)
        thr = (cs - stride - 1) / self.f
        n_cand = n_candidates(self.W, self.H, cs, stride)
        self.stats.update(h2d_bytes=0, d2h_bytes=0, launches=0, kernel_ms=0.0)
        L = lib()
        pending = []
        with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
            for ci, (e0, e1) in enumerate(self.chunks):
                d = self._static(ci)
                t = self._table(ci, n_cand, thr)
                counts = torch.empty(max(len(t), 1), dtype=torch.int32, device=self.device)
                d_t = torch.from_numpy(t).to(self.device)
                ev = self._events()
                check(L.sniper_chip_plan_count(d_t.data_ptr(), t.ctypes.data, len(t), S, cs, stride,
                                               d["box_off"].data_ptr(), d["wh"].data_ptr(), d["gt"].data_ptr(),
                                               counts.data_ptr(), self.stream.cuda_stream))
                ev[1].record(self.stream)
                self.stats["launches"] += 1
                nbox = counts.cpu().numpy()[:len(t)].astype(np.int64)
                self.stats["kernel_ms"] += ev[0].elapsed_time(ev[1])
                res = self._cover_assign(t, d, nbox, 0, None)
                xyxy, scale, first = self._chips(ci, res)
                local, cnt = self._lists(ci, res["owner"], first, len(xyxy))
                props = np.split(local.astype(np.int32), np.cumsum(cnt)[:-1]) if len(cnt) else []
                per_entry = first[::S]
                for k, e in enumerate(range(e0, e1)):
                    r = roidb[e]
                    lo, hi = per_entry[k], per_entry[k + 1]
                    tg = self.tags[e]
                    r['crops'] = [[xyxy[j]] + tg[scale[j]] for j in range(lo, hi)]
                    r['props_in_chips'] = props[lo:hi]
                if self.use_neg:
                    pending.append((t, res["owner_dev"], res["left"].astype(np.int64)))
            for ci, (t, pos_owner, left) in enumerate(pending):
                e0, e1 = self.chunks[ci]
                d = self._static(ci)
                res = self._cover_assign(t, d, left, 1, pos_owner)
                pending[ci] = None
                xyxy, scale, first = self._chips(ci, res)
                local, cnt = self._lists(ci, res["owner"], first, len(xyxy))
                keep = (cnt > 25) | ((cnt > 10) & (scale != 0))
                start = np.cumsum(cnt) - cnt
                per_entry = first[::S]
                ids = local.astype(np.int64)
                for k, e in enumerate(range(e0, e1)):
                    r = roidb[e]
                    tg = self.tags[e]
                    js = [j for j in range(per_entry[k], per_entry[k + 1]) if keep[j]]
                    r['neg_chips'] = r['neg_crops'] = [[xyxy[j]] + tg[scale[j]] for j in js]
                    r['neg_props_in_chips'] = [ids[start[j]:start[j] + cnt[j]].copy() for j in js]
        return roidb
