"""Argument validation of the depthwise weight gradient (csrc/depthwise.cu) and of the stream workspace registration
it shares with the wgmma weight gradient (csrc/capi_common.cu).

sniper_depthwise3x3_wgrad reads x and dy as 4-channel vectors, adds into dw, and sums its block partials in the slab of
the caller-owned workspace registered per (device, stream) with sniper_set_stream_workspace.  A bad shape, a null or
misaligned pointer, or a missing, null, misaligned or too small workspace must be refused BEFORE any CUDA call, with a
message naming the argument.  Every call below is built from fabricated, never dereferenced addresses and
violates exactly one rule.  On a machine without a device a check that wrongly passed would reach cudaGetDevice and
fail with a CUDA error instead of the expected message, so the message match also proves that no CUDA call was made.
There is deliberately no GPU variant of these tests."""
import re

import pytest

from sniper_b200 import _lib

A = 0x7f0000100000            # a fabricated 256-byte aligned address; never dereferenced
V = [A + 0x100000 * i for i in range(1, 6)]
ST = 0x7f00dead0000           # a fabricated stream handle with a registered (fabricated) workspace
ST_NONE = 0x7f00beef0000      # a fabricated stream handle nothing is registered for

WG = "x ldx dy lddy dw NB H W C stride dtype stream"
WG_GOOD = dict(x=A, ldx=64, dy=V[0], lddy=64, dw=V[1], NB=2, H=16, W=16, C=64, stride=1, dtype=1, stream=ST)
WS = "ws bytes device stream"


def _ws_bytes():
    return _lib.lib().sniper_stream_workspace_bytes()


def _call(name, order, args):
    L = _lib.lib()
    rc = getattr(L, name)(*[args[k] for k in order.split()])
    return rc, L.sniper_last_error().decode()


def _ws_good():
    return dict(ws=V[2], bytes=_ws_bytes(), device=0, stream=ST)


@pytest.fixture(scope="module", autouse=True)
def registered():
    """ST gets a (fabricated) workspace, so that the shape checks are reached with a workspace in place."""
    rc, msg = _call("sniper_set_stream_workspace", WS, _ws_good())
    assert rc == 0, msg


def _bad_wg(pattern, **change):
    a = dict(WG_GOOD)
    assert all(k in a for k in change)
    a.update(change)
    rc, msg = _call("sniper_depthwise3x3_wgrad", WG, a)
    assert rc == -1
    assert re.search(pattern, msg), msg


def _bad_ws(pattern, **change):
    a = _ws_good()
    assert all(k in a for k in change)
    a.update(change)
    rc, msg = _call("sniper_set_stream_workspace", WS, a)
    assert rc == -1
    assert re.search(pattern, msg), msg


def test_workspace_size_covers_a_full_wave_of_the_widest_blocks():
    # the fixed part, each region 256-byte aligned: split-K parked partials (132 tiles of 128 x 256 fp32), arrival
    # counters (132 x 8 ints), then the slab: 132 SMs x 4 blocks x 9 taps x 128 channels of fp32 partials
    assert _ws_bytes() == 132 * 128 * 256 * 4 + 4352 + 132 * 4 * 9 * 128 * 4


def test_registration_accepts_a_well_formed_workspace():
    rc, msg = _call("sniper_set_stream_workspace", WS, dict(_ws_good(), bytes=_ws_bytes() + 4096))
    assert rc == 0, msg
    rc, msg = _call("sniper_set_stream_workspace", WS, _ws_good())      # again: replaces the buffer
    assert rc == 0, msg


def test_null_workspace():
    _bad_ws(r"set_stream_workspace: ws must not be null", ws=0)


@pytest.mark.parametrize("off", [4, 8, 12, 16, 64, 128])
def test_misaligned_workspace(off):
    _bad_ws(r"set_stream_workspace: ws must be 256-byte aligned", ws=V[2] + off)


def test_too_small_workspace():
    n = _ws_bytes()
    _bad_ws(r"set_stream_workspace: bytes \(%d\) is smaller than sniper_stream_workspace_bytes\(\) \(%d\)" % (n - 4, n),
            bytes=n - 4)
    _bad_ws(r"set_stream_workspace: bytes \(0\) is smaller", bytes=0)


def test_negative_device():
    _bad_ws(r"set_stream_workspace: device \(-1\) must be >= 0", device=-1)


def test_no_workspace_for_the_stream():
    _bad_wg(r"depthwise3x3_wgrad: no workspace registered for this stream \(sniper_set_stream_workspace\)",
            stream=ST_NONE)


@pytest.mark.parametrize("dtype", [-1, 2])
def test_dtype(dtype):
    _bad_wg(r"depthwise3x3_wgrad: dtype \(%d\) must be 0 \(fp32\) or 1 \(bf16\)" % dtype, dtype=dtype)


@pytest.mark.parametrize("stride", [0, 3, -1])
def test_stride(stride):
    _bad_wg(r"depthwise3x3_wgrad: stride \(%d\) must be 1 or 2" % stride, stride=stride)


@pytest.mark.parametrize("arg", ["NB", "H", "W"])
@pytest.mark.parametrize("v", [0, -3])
def test_empty_or_negative_map(arg, v):
    _bad_wg(r"depthwise3x3_wgrad: NB \(-?\d+\), H \(-?\d+\) and W \(-?\d+\) must be positive", **{arg: v})


@pytest.mark.parametrize("C", [0, -4, 62])
def test_channels(C):
    _bad_wg(r"depthwise3x3_wgrad: C \(%d\) must be a positive multiple of 4" % C, C=C)


def test_channels_beyond_the_workspace():
    C = 132 * 4 * 128 + 4                        # 9 C partials no longer fit one slab row
    _bad_wg(r"depthwise3x3_wgrad: C \(%d\) exceeds the workspace's 67584 channels" % C, C=C, ldx=C, lddy=C)


@pytest.mark.parametrize("arg", ["ldx", "lddy"])
@pytest.mark.parametrize("v", [60, 66])
def test_pixel_strides(arg, v):
    _bad_wg(r"depthwise3x3_wgrad: %s \(%d\) must be a multiple of 4 and >= C \(64\)" % (arg, v), **{arg: v})


@pytest.mark.parametrize("arg", ["x", "dy", "dw"])
def test_null_pointers(arg):
    _bad_wg(r"depthwise3x3_wgrad: %s must not be null" % arg, **{arg: 0})


@pytest.mark.parametrize("arg", ["x", "dy"])
@pytest.mark.parametrize("dtype,off,need", [(0, 8, 16), (0, 4, 16), (1, 4, 8), (1, 2, 8)])
def test_misaligned_inputs(arg, dtype, off, need):
    _bad_wg(r"depthwise3x3_wgrad: %s must be %d-byte aligned" % (arg, need), dtype=dtype, **{arg: WG_GOOD[arg] + off})


def test_misaligned_dw():
    _bad_wg(r"depthwise3x3_wgrad: dw must be 4-byte aligned", dw=V[1] + 2)
