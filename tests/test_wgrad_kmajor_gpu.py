"""The tf32 weight gradient's channel-major operand copies (csrc/gemm_tc.cu, WgradFeed) on the device.

For stride-1 layers with several taps over rows of Wo % 32 == 0 pixels, sniper_conv2d_wgrad_nhwc copies dY and X
channel-major into the copy area of the workspace registered per (device, stream) and runs the K-major wgmma mainloop
on the copies; other tf32 layers transpose in the kernel.  What the exact table of test_gemm_exact_gpu.py cannot see:
  * the copy area grows on a stream, and a graph captured on another stream (whose workspace is allocated during the
    capture) replays to the same bytes as eager calls;
  * a tf32 call on a stream without a workspace, or with too small a copy area, is refused before any launch;
  * the step's own geometries at 2 chips, bit for bit against float64 on integer operands: the 3 x 3 layer over 3072
    channels at 32 x 32 (the RPN conv, from copies), and the transposing path's 3 x 3 stride-2 layer at 128 -> 64 and
    1 x 1 stride-2 shortcut.
"""
import ctypes

import numpy as np
import pytest
import torch

from sniper_b200 import _lib, ops

pytestmark = pytest.mark.gpu


def _ints(*shape, gen):
    return torch.randint(-1, 2, shape, generator=gen, dtype=torch.int32).float().cuda()


def _reference(dy, x, k, stride, dil, pad):
    """dW[Cout, (kh, kw, ci)] in float64"""
    Cout, Cin = dy.shape[3], x.shape[3]
    xn = x.double().permute(0, 3, 1, 2)
    dyn = dy.double().permute(0, 3, 1, 2)
    w = torch.nn.grad.conv2d_weight(xn, (Cout, Cin, k, k), dyn, stride=stride, padding=pad, dilation=dil)
    return w.permute(0, 2, 3, 1).reshape(Cout, k * k * Cin)


@pytest.mark.parametrize("NB,H,Cin,Cout,k,stride,dil,pad", [
    (2, 128, 128, 128, 3, 2, 1, 1),      # stage-2 unit-1 conv2: 128 -> 64, transposed in the kernel
    (2, 128, 256, 512, 1, 2, 1, 0),      # stage-2 unit-1 shortcut: 1 x 1 stride 2, transposed in the kernel
    (2, 32, 3072, 512, 3, 1, 1, 1),      # rpn_conv_3x3: 3072 channels at 32 x 32, from copies
], ids=["conv2_s2_128to64", "sc_1x1_s2", "rpn_3x3_c3072"])
def test_step_geometry_is_integer_exact(NB, H, Cin, Cout, k, stride, dil, pad):
    gen = torch.Generator().manual_seed(Cin + 7 * Cout + stride)
    Ho = (H + 2 * pad - dil * (k - 1) - 1) // stride + 1
    x = _ints(NB, H, H, Cin, gen=gen)
    dy = _ints(NB, Ho, Ho, Cout, gen=gen)
    ref = _reference(dy, x, k, stride, dil, pad)
    assert ref.abs().max().item() < 2 ** 24
    for splits in (1, 0):
        dw = ops.conv2d_wgrad_nhwc(dy, x, kh=k, kw=k, stride=stride, dil=dil, pad=pad, splits=splits)
        torch.cuda.synchronize()
        assert torch.equal(dw.double(), ref), (splits, (dw.double() - ref).abs().max().item())


def _fresh_workspace(stream):
    """torch hands out pool streams round-robin, so `stream` may be a handle an earlier test grew a workspace on: retire
    that workspace (kept alive like a replaced one), so that the next call on the stream allocates afresh"""
    key = (torch.cuda.current_device(), stream.cuda_stream)
    if key in ops._workspaces:
        ops._replaced_workspaces.append(ops._workspaces.pop(key))


def test_scratch_growth_and_graph_replay_on_another_stream():
    gen = torch.Generator().manual_seed(5)
    small_x, small_dy = torch.randn(1, 4, 32, 64, generator=gen).cuda(), torch.randn(1, 4, 32, 64, generator=gen).cuda()
    x, dy = torch.randn(2, 64, 64, 256, generator=gen).cuda(), torch.randn(2, 64, 64, 128, generator=gen).cuda()
    args = dict(kh=3, kw=3, pad=1, splits=4)
    s1 = torch.cuda.Stream()
    _fresh_workspace(s1)
    s1.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s1):
        ops.conv2d_wgrad_nhwc(small_dy, small_x, **args)
        n_small = ops._stream_workspace().numel()
        eager = ops.conv2d_wgrad_nhwc(dy, x, **args)          # needs more: the stream's workspace grows
        assert ops._stream_workspace().numel() > n_small
        eager2 = ops.conv2d_wgrad_nhwc(dy, x, **args)
    torch.cuda.current_stream().wait_stream(s1)
    torch.cuda.synchronize()
    assert torch.equal(eager, eager2)
    ref = _reference(dy, x, 3, 1, 1, 1)
    assert (eager.double() - ref).abs().max().item() < 1e-2 * ref.abs().max().item()

    dw = torch.zeros_like(eager)
    s2 = torch.cuda.Stream()
    _fresh_workspace(s2)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s2):
        dw.zero_()
        ops.conv2d_wgrad_nhwc(dy, x, dw_out=dw, **args)
    for _ in range(2):
        dw.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(dw, eager)


def _raw_wgrad(dy, x, dw, stream):
    dh, dw_ = ops.conv_taps(3, 3, 1, 1)
    a = np.ascontiguousarray(dh, dtype=np.int32)
    b = np.ascontiguousarray(dw_, dtype=np.int32)
    NB, H, W, Cin = x.shape
    Cout = dy.shape[3]
    L = _lib.lib()
    rc = L.sniper_conv2d_wgrad_nhwc(dy.data_ptr(), Cout, x.data_ptr(), Cin, NB, H, W, Cin, Cout, 9,
                                    a.ctypes.data_as(ctypes.c_void_p), b.ctypes.data_as(ctypes.c_void_p), 1, H, W,
                                    dw.data_ptr(), 0, 1, stream)
    return rc, L.sniper_last_error().decode()


def test_tf32_call_without_scratch_is_refused():
    """Fabricated stream handles (never registered by ops, never enqueued on): the refusal comes before any launch."""
    x, dy = torch.ones(1, 32, 32, 64, device="cuda"), torch.ones(1, 32, 32, 64, device="cuda")
    dw = torch.zeros(64, 9 * 64, device="cuda")
    rc, err = _raw_wgrad(dy, x, dw, 0x7f00beef0000)
    assert rc != 0 and "no workspace registered for this stream (sniper_set_stream_workspace)" in err, err
    L = _lib.lib()
    buf = torch.zeros(L.sniper_stream_workspace_bytes() + (1 << 16), dtype=torch.uint8, device="cuda")
    _lib.check(L.sniper_set_stream_workspace(buf.data_ptr(), buf.numel(), torch.cuda.current_device(), 0x7f00beef1000))
    rc, err = _raw_wgrad(dy, x, dw, 0x7f00beef1000)
    assert rc != 0 and "65536-byte copy area, this call needs" in err, err
    torch.cuda.synchronize()
    assert not dw.any().item()
