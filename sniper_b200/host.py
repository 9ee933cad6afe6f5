"""Host-side members of the path (numpy in / numpy out) over the C-ABI: chip sampling, NMS, overlaps.
Mirrors lib/chips/chips.pyx, lib/nms/nms.py and lib/bbox of the reference (chip_generator / chip_worker: chip_worker.py),
and the image reader the reference takes from OpenCV (`imread`, on PIL)."""
import ctypes

import numpy as np

from ._lib import check, lib

_libc = ctypes.CDLL(None)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def srand(seed):
    """Seeds the C rand() stream chips_generate draws from (the reference never seeds: glibc default = 1)."""
    _libc.srand(ctypes.c_uint(seed))


def chips_generate(boxes, width, height, chipsize, stride):
    """chips.generate(boxes f32[N,4], w, h, chipsize, stride) (lib/chips/chips.pyx:16-21) -> [n,4] float32."""
    boxes = np.ascontiguousarray(boxes, dtype=np.float32).reshape(-1, 4)
    out = np.zeros((4096, 4), np.float32)
    n = lib().sniper_chips_generate(_p(boxes), boxes.shape[0], int(width), int(height), int(chipsize), int(stride),
                                    _p(out), 4096)
    if n < 0:
        check(-1)
    return out[:n].copy()


def cpu_nms(dets, thresh, order=None):
    """cpu_nms(dets f32[N,5], thresh) (lib/nms/cpu_nms.pyx:112-163) -> keep indices (list)."""
    dets = np.ascontiguousarray(dets, dtype=np.float32)
    n = dets.shape[0]
    if order is None:
        order = dets[:, 4].argsort()[::-1]
    order = np.ascontiguousarray(order, dtype=np.int64)
    keep = np.zeros((max(n, 1),), np.int32)
    k = lib().sniper_cpu_nms(_p(dets), _p(order), n, float(thresh), _p(keep))
    return keep[:k].tolist()


def cpu_soft_nms(boxes, sigma=0.5, Nt=0.3, threshold=0.001, method=2):
    """cpu_soft_nms (lib/nms/cpu_nms.pyx:17-110): returns the surviving rows (scores decayed), boxes is modified."""
    assert boxes.dtype == np.float32 and boxes.flags.c_contiguous
    n = lib().sniper_cpu_soft_nms(_p(boxes), boxes.shape[0], float(sigma), float(Nt), float(threshold), int(method))
    return boxes[:n, :]


def bbox_overlaps(boxes, query_boxes):
    b = np.ascontiguousarray(boxes, dtype=np.float64)
    q = np.ascontiguousarray(query_boxes, dtype=np.float64)
    out = np.zeros((b.shape[0], q.shape[0]), np.float64)
    check(lib().sniper_bbox_overlaps(_p(b), b.shape[0], _p(q), q.shape[0], _p(out), 0))
    return out


def ignore_overlaps(boxes, query_boxes):
    b = np.ascontiguousarray(boxes, dtype=np.float64)
    q = np.ascontiguousarray(query_boxes, dtype=np.float64)
    out = np.zeros((b.shape[0], q.shape[0]), np.float64)
    check(lib().sniper_bbox_overlaps(_p(b), b.shape[0], _p(q), q.shape[0], _p(out), 1))
    return out


def imread(path):
    """cv2.imread(path, cv2.IMREAD_COLOR) on PIL: uint8 [H, W, 3] in BGR order.  Grayscale and palette images are
    expanded to three channels, an alpha channel is dropped and the EXIF orientation is applied.  Raises OSError
    naming the path when the file cannot be read or decoded (cv2.imread would return None)."""
    try:
        from PIL import Image, ImageOps
    except ImportError as e:
        raise ImportError("host.imread decodes images with Pillow (PIL), which is not installed") from e
    try:
        with Image.open(path) as im:
            rgb = np.asarray(ImageOps.exif_transpose(im).convert('RGB'))
    except OSError as e:
        raise OSError("imread: cannot read image %s: %s" % (path, e)) from e
    return np.ascontiguousarray(rgb[:, :, ::-1])
