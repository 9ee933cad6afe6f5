"""MXNet `.params` wire format + the name / layout mapping between the reference's checkpoints and this repo's tensors.

File format (SNIPER-mxnet/src/ndarray/ndarray.cc:1547-1790, NDArray::Save / Load and the list form used by
`mx.nd.save` / `mx.model.save_checkpoint`; keys are "arg:<name>" / "aux:<name>", lib/train_utils/utils.py:45-65):

    uint64 0x112 | uint64 0 | uint64 n | n x NDArray | uint64 n_names | n_names x (uint64 len | bytes)
    NDArray v2 : uint32 0xF993fac9 | int32 stype (0 = dense) | shape | int32 dev_type | int32 dev_id | int32 type_flag | data
    NDArray v1 : uint32 0xF993fac8 | shape | ctx | type_flag | data          legacy: uint32 ndim | uint32 dims[ndim] | ...
    shape      : uint32 ndim | int64 dims[ndim]                                  (nnvm/tuple.h:553-579, dim_t = int64)
    type_flag  : 0 f32, 1 f64, 2 f16, 3 u8, 4 i32, 5 i8, 6 i64                    (mshadow/base.h:295-301)

Layouts: the reference stores convolution weights OIHW and FullyConnected weights [out, C*H*W] over NCHW inputs; this
repo runs NHWC implicit GEMMs, i.e. rows [O, kh*kw*I] (tap-major, channel-minor) and FC inputs flattened (h, w, c).
`rpn_head` = rpn_bbox_pred (4A rows) followed by rpn_cls_score (2A rows); `cls_bbox` = cls_score (K rows) followed by
bbox_pred (4 rows); output rows are zero-padded to the tile-friendly counts the kernels use."""
import struct

import numpy as np
import torch

LIST_MAGIC = 0x112
V1_MAGIC = 0xF993FAC8
V2_MAGIC = 0xF993FAC9
_DTYPES = {0: np.float32, 1: np.float64, 2: np.float16, 3: np.uint8, 4: np.int32, 5: np.int8, 6: np.int64}
_FLAGS = {np.dtype(v): k for k, v in _DTYPES.items()}


class _Reader:
    def __init__(self, buf):
        self.b, self.o = buf, 0

    def take(self, fmt):
        v = struct.unpack_from("<" + fmt, self.b, self.o)
        self.o += struct.calcsize("<" + fmt)
        return v if len(v) > 1 else v[0]

    def raw(self, n):
        v = self.b[self.o:self.o + n]
        if len(v) != n:
            raise ValueError("truncated .params file")
        self.o += n
        return v


def _read_ndarray(r):
    magic = r.take("I")
    if magic == V2_MAGIC:
        stype = r.take("i")
        if stype != 0:
            raise ValueError("sparse NDArray (stype %d) is not supported" % stype)
        ndim = r.take("I")
        shape = [r.take("q") for _ in range(ndim)]
    elif magic == V1_MAGIC:
        ndim = r.take("I")
        shape = [r.take("q") for _ in range(ndim)]
    else:                                   # legacy: the magic word is ndim, dims are uint32
        ndim = magic
        shape = [r.take("I") for _ in range(ndim)]
    if ndim == 0:
        return None
    r.take("ii")                            # context (dev_type, dev_id): everything is loaded to host memory
    flag = r.take("i")
    dt = np.dtype(_DTYPES[flag])
    n = int(np.prod(shape))
    return np.frombuffer(r.raw(n * dt.itemsize), dtype=dt).reshape(shape).copy()


def read_list(path):
    """`mx.nd.load` of a named NDArray list -> [(name, numpy array)] in file order."""
    r = _Reader(open(path, "rb").read())
    if r.take("Q") != LIST_MAGIC:
        raise ValueError("%s is not an MXNet NDArray list file" % path)
    r.take("Q")
    arrays = [_read_ndarray(r) for _ in range(r.take("Q"))]
    names = [r.raw(r.take("Q")).decode() for _ in range(r.take("Q"))]
    if len(names) != len(arrays):
        raise ValueError("unnamed NDArray lists are not checkpoints")
    return list(zip(names, arrays))


def read_params(path):
    """`mx.nd.load` + the arg:/aux: split of load_checkpoint (utils.py:56-65) -> (arg_params, aux_params) as numpy."""
    arg, aux = {}, {}
    for k, v in read_list(path):
        tp, name = k.split(":", 1)
        (arg if tp == "arg" else aux)[name] = v
    return arg, aux


def write_params(path, arg, aux):
    """`mx.model.save_checkpoint`'s `.params` half (NDArray v2, dense, cpu context)."""
    write_list(path, [("arg:" + k, v) for k, v in arg.items()] + [("aux:" + k, v) for k, v in aux.items()])


def write_list(path, items):
    """`mx.nd.save` of a named NDArray list [(name, numpy array)]."""
    out = [struct.pack("<QQQ", LIST_MAGIC, 0, len(items))]
    for _, v in items:
        v = np.ascontiguousarray(v)
        out.append(struct.pack("<Ii", V2_MAGIC, 0))
        out.append(struct.pack("<I", v.ndim) + struct.pack("<%dq" % v.ndim, *v.shape))
        out.append(struct.pack("<iii", 1, 0, _FLAGS[v.dtype]))
        out.append(v.tobytes())
    out.append(struct.pack("<Q", len(items)))
    for k, _ in items:
        kb = k.encode()
        out.append(struct.pack("<Q", len(kb)) + kb)
    with open(path, "wb") as f:
        f.write(b"".join(out))


BBOX_STDS_TEST = (0.1, 0.1, 0.2, 0.2)      # hard-coded in the reference's checkpoint_callback (resnet_mx_101_e2e.py:11)


def save_checkpoint(prefix, epoch, arg, aux, bbox_param_names=("bbox_pred_weight", "bbox_pred_bias")):
    """`checkpoint_callback` (symbols/faster/resnet_mx_101_e2e.py:6-17) + the `.params` half of
    mx.model.save_checkpoint: writes `<prefix>-%04d.params` with the extra `*_test` copies of the box-regression layer
    (weight rows and bias scaled by the target stds, what the test-time symbol binds).  Returns the path."""
    out = dict(arg)
    if bbox_param_names[0] in arg:
        stds = np.array(BBOX_STDS_TEST, dtype=arg[bbox_param_names[0]].dtype)
        out[bbox_param_names[0] + "_test"] = (arg[bbox_param_names[0]].T * stds).T
        out[bbox_param_names[1] + "_test"] = arg[bbox_param_names[1]] * stds
    path = "%s-%04d.params" % (prefix, epoch)
    write_params(path, out, aux)
    return path


def load_param(prefix, epoch, process=False):
    """lib/train_utils/utils.py:77-100: (arg_params, aux_params) of `<prefix>-%04d.params`; process=True renames the
    `*_test` tensors over the training ones (what main_test.py loads)."""
    arg, aux = read_params("%s-%04d.params" % (prefix, epoch))
    if process:
        for k in [k for k in arg if "_test" in k]:
            arg[k.replace("_test", "")] = arg.pop(k)
    return arg, aux


# ---------------------------------------------------------------------------------------------------------------
# layout conversions (numpy, pure functions)
# ---------------------------------------------------------------------------------------------------------------
def conv_to_rows(w_oihw, rows=None):
    """OIHW -> [O(+pad), kh*kw*I] (tap-major, channel-minor)."""
    O, I, kh, kw = w_oihw.shape
    m = np.ascontiguousarray(w_oihw.transpose(0, 2, 3, 1)).reshape(O, kh * kw * I)
    return pad_rows(m, rows)


def rows_to_conv(m, O, I, k):
    return np.ascontiguousarray(m[:O].reshape(O, k, k, I).transpose(0, 3, 1, 2))


def fc_chw_to_hwc(w, C, H, W, rows=None):
    """FullyConnected weight over an NCHW-flattened input -> the same map over an NHWC-flattened input."""
    O = w.shape[0]
    m = np.ascontiguousarray(w.reshape(O, C, H, W).transpose(0, 2, 3, 1)).reshape(O, H * W * C)
    return pad_rows(m, rows)


def fc_hwc_to_chw(m, O, C, H, W):
    return np.ascontiguousarray(m[:O].reshape(O, H, W, C).transpose(0, 3, 1, 2)).reshape(O, C * H * W)


def pad_rows(m, rows):
    if rows is None or rows == m.shape[0]:
        return m
    out = np.zeros((rows,) + m.shape[1:], m.dtype)
    out[:m.shape[0]] = m
    return out


def fuse_rows(parts, rows=None):
    return pad_rows(np.concatenate(parts, 0), rows)


# ---------------------------------------------------------------------------------------------------------------
# the network-level mapping (names of symbols/faster/resnet_mx_101_e2e.py <-> model.SniperResNet101)
# ---------------------------------------------------------------------------------------------------------------
FUSED = {   # our fused tensor -> reference parts in row order
    "rpn_head": ("rpn_bbox_pred", "rpn_cls_score"),
    "cls_bbox": ("cls_score", "bbox_pred"),
}
FC_OVER_POOLED = {"offset": (256, 7, 7), "fc_new_1": (256, 7, 7)}   # FCs that read the 7x7x256 pooled features
FC_PLAIN = ("fc_new_2", "cls_score", "bbox_pred")                     # FullyConnected layers with 2-D weights


def conv_from_reference(name, cout, coutp, cin, k, bias, arg):
    """Reference tensors of layer `name` -> (rows [coutp, k*k*cin], bias [coutp] or None) in this repo's layout."""
    def one(n):
        w = arg[n + "_weight"]
        if n in FC_OVER_POOLED and w.ndim == 2:
            m = fc_chw_to_hwc(w, *FC_OVER_POOLED[n])
        elif w.ndim == 2:
            m = w
        else:
            m = conv_to_rows(w)
        return m, (arg[n + "_bias"] if bias else None)
    parts = [one(n) for n in FUSED.get(name, (name,))]
    w = fuse_rows([p[0] for p in parts], coutp).astype(np.float32)
    if w.shape != (coutp, k * k * cin) or sum(p[0].shape[0] for p in parts) != cout:
        raise ValueError("checkpoint tensor(s) of %s have shape %s, expected %d x %d" % (name, w.shape, cout, k * k * cin))
    b = fuse_rows([p[1] for p in parts], coutp).astype(np.float32) if bias else None
    return w, b


def conv_to_reference(name, cout, cin, k, w_rows, b, part_rows=None, out=None):
    """Inverse of conv_from_reference: fills `out` (arg dict) with the reference tensors of layer `name`.
    part_rows: row counts of the fused parts (FUSED layers)."""
    out = {} if out is None else out
    parts = FUSED.get(name, (name,))
    counts = part_rows if part_rows is not None else [cout]
    r0 = 0
    for n, c in zip(parts, counts):
        m = w_rows[r0:r0 + c]
        if n in FC_OVER_POOLED:
            out[n + "_weight"] = fc_hwc_to_chw(m, c, *FC_OVER_POOLED[n])
        elif n in FC_PLAIN:
            out[n + "_weight"] = np.ascontiguousarray(m)
        else:
            out[n + "_weight"] = rows_to_conv(m, c, cin, k)
        if b is not None:
            out[n + "_bias"] = np.ascontiguousarray(b[r0:r0 + c])
        r0 += c
    return out


# ---------------------------------------------------------------------------------------------------------------
# optimizer state (`<prefix>-%04d.states`)
# ---------------------------------------------------------------------------------------------------------------
def _momentum_index(net):
    """For every trainable tensor of net.export_reference(grads=True) (reference name and layout): the flat position of
    each element in net.P.  Found by exporting an index image of the gradient buffer (two halves, each exact in float32)
    and restoring the buffer afterwards, so the momenta go through exactly the conversions the weights go through."""
    P = net.P
    saved = P.g.clone()
    idx = torch.arange(P.total, device=P.g.device)
    parts = []
    try:
        for v in (idx % 4096, idx // 4096):
            P.g.copy_(v.float())
            parts.append(net.export_reference(grads=True)[0])
    finally:
        P.g.copy_(saved)
    return {k: parts[0][k].astype(np.int64) + 4096 * parts[1][k].astype(np.int64) for k in parts[0]}


def save_optimizer_states(path, net, num_update):
    """The SGD state a stopped run needs: the momentum of every trainable tensor as `mom:<reference name>` in the
    reference's layout, and the update count as int64 `num_update`, in the NDArray-list format of `.params` files.
    (MXNet's own `.states` is a pickled Updater.states dict, optimizer.py:1487-1505: the two are not interchangeable.)"""
    mom = net.P.mom.detach().cpu().numpy()
    items = [("mom:" + k, np.ascontiguousarray(mom[v])) for k, v in _momentum_index(net).items()]
    items.append(("num_update", np.array([int(num_update)], dtype=np.int64)))
    write_list(path, items)
    return path


def load_optimizer_states(path, net):
    """Inverse of save_optimizer_states: fills net.P.mom and returns num_update."""
    items = dict(read_list(path))
    mom = np.zeros(net.P.total, dtype=np.float32)
    for k, v in _momentum_index(net).items():
        m = items.get("mom:" + k)
        if m is None or m.shape != v.shape:
            raise ValueError("%s: no momentum of shape %s for %s" % (path, v.shape, k))
        mom[v] = m
    if "num_update" not in items:
        raise ValueError("%s has no num_update" % path)
    net.P.mom.copy_(torch.from_numpy(mom))
    return int(items["num_update"].reshape(-1)[0])
