"""Argument validation of the depthwise forward, its data gradient and the first-layer im2col (csrc/depthwise.cu).

sniper_depthwise3x3_fwd / _dgrad read and write the maps as 4-channel vectors (16 bytes of fp32, 8 bytes of bf16) and
the weights [9, C] as float4; sniper_im2col3x3s2_nchw reads the fp32 image by element and stores 4 columns at a time.
A bad shape, or a null or misaligned pointer, must be refused BEFORE any CUDA call, with a message naming the argument.
Every call below is built from fabricated, never dereferenced addresses and violates exactly one rule.  On a machine
without a device a check that wrongly passed would reach the kernel launch and fail with a CUDA error instead of the
expected message, so the message match also proves that no CUDA call was made.  No call here is well formed: which
kernel a well-formed call picks (tiled or register) is checked on the device by tests/test_dw_exact_gpu.py."""
import re

import pytest

from sniper_b200 import _lib

A = 0x7f0000100000            # a fabricated 256-byte aligned address; never dereferenced
V = [A + 0x100000 * i for i in range(1, 4)]
ST = 0x7f00dead0000           # a fabricated stream handle

DW = {"fwd": ("sniper_depthwise3x3_fwd", "x ldx w y ldy NB H W C stride dtype stream", "x", "y"),
      "dgrad": ("sniper_depthwise3x3_dgrad", "dy lddy w dx lddx NB H W C stride dtype stream", "dy", "dx")}
IC = "x col NB H W Cin Kp dtype stream"
IC_GOOD = dict(x=A, col=V[0], NB=2, H=16, W=16, Cin=3, Kp=64, dtype=1, stream=ST)


def _dw_good(op, stride=1, dtype=1):
    _, order, i, o = DW[op]
    ld_i, ld_o = order.split()[1], order.split()[4]
    return {i: A, ld_i: 64, "w": V[0], o: V[1], ld_o: 64, "NB": 2, "H": 16, "W": 16, "C": 64, "stride": stride,
            "dtype": dtype, "stream": ST}


def _call(name, order, args):
    L = _lib.lib()
    rc = getattr(L, name)(*[args[k] for k in order.split()])
    return rc, L.sniper_last_error().decode()


def _bad(name, order, good, pattern, change):
    a = dict(good)
    assert all(k in a for k in change)
    a.update(change)
    rc, msg = _call(name, order, a)
    assert rc == -1
    assert re.search(pattern, msg), msg


def _bad_dw(op, pattern, stride=1, dtype=1, **change):
    name, order, _, _ = DW[op]
    _bad(name, order, _dw_good(op, stride, dtype), r"depthwise3x3_%s: " % op + pattern, change)


def _bad_ic(pattern, **change):
    _bad("sniper_im2col3x3s2_nchw", IC, IC_GOOD, r"im2col3x3s2: " + pattern, change)


OPS = ["fwd", "dgrad"]
STRIDES = [1, 2]                # the data gradient checks its pointers on both of its branches


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("dtype", [-1, 2])
def test_dtype(op, dtype):
    _bad_dw(op, r"dtype must be 0 \(fp32\) or 1 \(bf16\)", dtype=dtype)


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("stride", [0, 3, -1])
def test_stride(op, stride):
    _bad_dw(op, r"stride must be 1 or 2", stride=stride)


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("arg", ["NB", "H", "W"])
@pytest.mark.parametrize("v", [0, -3])
def test_empty_or_negative_map(op, arg, v):
    _bad_dw(op, r"NB \(-?\d+\), H \(-?\d+\) and W \(-?\d+\) must be positive", **{arg: v})


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("C", [0, -4, 62])
def test_channels(op, C):
    _bad_dw(op, r"C \(%d\) must be a positive multiple of 4" % C, C=C)


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("stride", STRIDES)
@pytest.mark.parametrize("which", [1, 4])
@pytest.mark.parametrize("v", [60, 66])
def test_pixel_strides(op, stride, which, v):
    ld = DW[op][1].split()[which]
    _bad_dw(op, r"pixel strides must be multiples of 4 and >= C", stride=stride, **{ld: v})


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("stride", STRIDES)
@pytest.mark.parametrize("which", ["in", "w", "out"])
def test_null_pointers(op, stride, which):
    arg = {"in": DW[op][2], "w": "w", "out": DW[op][3]}[which]
    _bad_dw(op, r"%s must not be null" % arg, stride=stride, **{arg: 0})


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("stride", STRIDES)
@pytest.mark.parametrize("which", ["in", "out"])
@pytest.mark.parametrize("dtype,off,need", [(0, 4, 16), (0, 8, 16), (0, 12, 16), (1, 2, 8), (1, 4, 8), (1, 6, 8)])
def test_misaligned_maps(op, stride, which, dtype, off, need):
    arg = DW[op][2] if which == "in" else DW[op][3]
    good = _dw_good(op, stride, dtype)
    _bad_dw(op, r"%s must be %d-byte aligned" % (arg, need), stride=stride, dtype=dtype, **{arg: good[arg] + off})


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("stride", STRIDES)
@pytest.mark.parametrize("dtype", [0, 1])
@pytest.mark.parametrize("off", [4, 8, 12])
def test_misaligned_weights(op, stride, dtype, off):
    _bad_dw(op, r"w must be 16-byte aligned", stride=stride, dtype=dtype, w=V[0] + off)


def test_im2col_dtype():
    _bad_ic(r"dtype must be 0 \(fp32\) or 1 \(bf16\)", dtype=2)


def test_im2col_channels():
    _bad_ic(r"built for the 3-channel first layer \(Cin = 4\)", Cin=4)


@pytest.mark.parametrize("Kp", [26, 30, 0])
def test_im2col_columns(Kp):
    _bad_ic(r"Kp \(%d\) must be a multiple of 4 and >= 27" % Kp, Kp=Kp)


@pytest.mark.parametrize("arg", ["NB", "H", "W"])
def test_im2col_empty(arg):
    _bad_ic(r"empty input", **{arg: 0})


@pytest.mark.parametrize("arg", ["x", "col"])
def test_im2col_null_pointers(arg):
    _bad_ic(r"%s must not be null" % arg, **{arg: 0})


@pytest.mark.parametrize("off", [1, 2, 3])
def test_im2col_misaligned_image(off):
    _bad_ic(r"x must be 4-byte aligned", x=A + off)


@pytest.mark.parametrize("dtype,off,need", [(0, 4, 16), (0, 8, 16), (0, 12, 16), (1, 2, 8), (1, 4, 8), (1, 6, 8)])
def test_im2col_misaligned_columns(dtype, off, need):
    _bad_ic(r"col must be %d-byte aligned" % need, dtype=dtype, col=V[0] + off)


def test_pixel_stride_of_channel_slices_and_size_one_dims():
    """The wrappers pass ops._pixel_ld as ldx / ldy: the pixel stride of a channel slice, with the strides of size-1
    dimensions (which no kernel uses) not checked, as for the convolution weight gradient that shares the helper."""
    import torch
    from sniper_b200 import ops
    assert ops._pixel_ld(torch.zeros(2, 5, 7, 128)[..., 4:68]) == 128
    assert ops._pixel_ld(torch.zeros(1, 8, 8, 64)[:, :4]) == 64
    assert ops._pixel_ld(torch.zeros(3, 1, 9, 68)[..., :64]) == 68
    with pytest.raises(AssertionError):
        ops._pixel_ld(torch.zeros(2, 8, 8, 64)[:, :4])          # the images no longer follow each other
    with pytest.raises(AssertionError):
        ops._pixel_ld(torch.zeros(2, 8, 64, 8).transpose(2, 3))   # channels not contiguous
