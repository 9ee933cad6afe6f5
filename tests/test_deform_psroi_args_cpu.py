"""Argument validation of the deformable-convolution and (Deformable)PSROIPooling entry points (csrc/deform_conv.cu,
csrc/psroi.cu).

The deformable im2col / col2im warps read x and write col as whole 16-byte (fp32) or 8-byte (bf16) vectors, scatter dx
with float4 atomics (sniper_deform_col2im) or double atomics into `acc` (sniper_deform_col2im_fp64acc), and divide by
the stride when they size the output map.  A misaligned pointer, a zero stride or a negative size must be refused
BEFORE any CUDA call, with a message naming the argument.  Every call below is built from fabricated, never dereferenced
addresses and violates exactly one rule, so it returns from its check; with NB == 0 / num_rois == 0 in place, even a
check that wrongly passed could not launch anything.  There is deliberately no GPU variant of these tests.  The empty
calls prove "no launch" the same way: they must return 0, which a launch attempt on a machine without a device could
not."""
import re

import pytest

from sniper_b200 import _lib

A = 0x7f0000100000            # a fabricated 256-byte aligned address; never dereferenced
V = [A + 0x100000 * i for i in range(1, 12)]     # distinct aligned addresses


def _call(name, args):
    L = _lib.lib()
    rc = getattr(L, name)(*args)
    return rc, L.sniper_last_error().decode()


_DC = "x offset NB H W C KH KW stride dil pad dgroups off_ld"
_DC_GOOD = dict(x=A, offset=V[0], NB=0, H=10, W=12, C=512, KH=3, KW=3, stride=1, dil=2, pad=2, dgroups=4, off_ld=96,
                dtype=0, stream=0)
_PS = ("num_rois channels height width spatial_scale output_dim group_size pooled_size part_size sample_per_part "
       "trans_std no_trans num_classes")
_PS_GOOD = dict(num_rois=0, channels=256, height=20, width=30, spatial_scale=0.0625, output_dim=256, group_size=1,
                pooled_size=7, part_size=7, sample_per_part=4, trans_std=0.1, no_trans=0, num_classes=1, layout=1,
                stream=0)

# name -> (argument names in ABI order, a well-formed empty call)
GOOD = {
    "sniper_deform_im2col": (_DC + " col dtype stream", dict(_DC_GOOD, col=V[1])),
    "sniper_deform_col2im": ("dcol " + _DC + " dx doffset dtype stream", dict(_DC_GOOD, dcol=V[1], dx=V[2], doffset=V[3])),
    "sniper_deform_col2im_fp64acc": ("dcol " + _DC + " dx doffset dtype acc acc_elems stream",
                                     dict(_DC_GOOD, dcol=V[1], dx=V[2], doffset=V[3], acc=V[4], acc_elems=0)),
    "sniper_deform_psroi_fwd": ("data rois trans " + _PS + " layout top_data top_count sample_idx stream",
                                dict(_PS_GOOD, data=A, rois=V[0], trans=V[1], top_data=V[2], top_count=V[3],
                                     sample_idx=0)),
    "sniper_deform_psroi_bwd": ("top_diff data rois trans " + _PS + " layout data_diff trans_diff stream",
                                dict(_PS_GOOD, top_diff=V[2], data=A, rois=V[0], trans=V[1], data_diff=V[4],
                                     trans_diff=V[5])),
    "sniper_deform_psroi_bwd_fp64acc": ("top_diff data rois trans num_rois batch " + _PS.split(" ", 1)[1] +
                                        " data_diff trans_diff acc acc_elems stream",
                                        dict(_PS_GOOD, top_diff=V[2], data=A, rois=V[0], trans=V[1], batch=2,
                                             data_diff=V[4], trans_diff=V[5], acc=V[6], acc_elems=2 * 20 * 30 * 256)),
    "sniper_psroi_fwd": ("data rois num_rois channels height width spatial_scale output_dim group_size pooled_size "
                         "layout top_data bins stream",
                         dict(_PS_GOOD, data=A, rois=V[0], channels=18, output_dim=2, group_size=3, pooled_size=3,
                              layout=0, top_data=V[2], bins=0)),
    "sniper_psroi_bwd": ("top_diff rois num_rois channels height width spatial_scale output_dim group_size pooled_size "
                         "layout data_diff stream",
                         dict(_PS_GOOD, top_diff=V[2], rois=V[0], channels=18, output_dim=2, group_size=3,
                              pooled_size=3, layout=0, data_diff=V[4])),
}
DC = [n for n in GOOD if "deform_col2im" in n or "deform_im2col" in n]
PS = [n for n in GOOD if n not in DC]


def _args(name, **change):
    order, good = GOOD[name]
    a = dict(good)
    for k in change:
        assert k in order.split(), (name, k)
    a.update(change)
    return [a[k] for k in order.split()]


@pytest.mark.parametrize("name", sorted(GOOD))
def test_empty_call_is_accepted_without_a_launch(name):
    rc, msg = _call(name, _args(name))
    assert rc == 0, msg


@pytest.mark.parametrize("dtype", [0, 1])
@pytest.mark.parametrize("name", sorted(DC))
def test_empty_deform_call_in_either_dtype(name, dtype):
    """NB == 0 with a kernel that fits the map, in both storage types, and with the padded-offset and exact-stride
    layouts: accepted, nothing launched."""
    for off_ld in (72, 96):
        rc, msg = _call(name, _args(name, dtype=dtype, off_ld=off_ld))
        assert rc == 0, msg


def test_empty_deform_call_needs_no_output_map():
    """NB == 0 is empty whatever the map: a kernel larger than the padded map is not an error then."""
    rc, msg = _call("sniper_deform_im2col", _args("sniper_deform_im2col", H=1, W=1, pad=0))
    assert rc == 0, msg


BAD = []


def _bad(name, pattern, **change):
    BAD.append(pytest.param(name, change, pattern, id="%s-%s" % (name[7:], "-".join(
        "%s=%s" % (k, "+%d" % (v - A) if isinstance(v, int) and v >= A else v) for k, v in change.items()))))


for name in DC:
    fn = name[7:]
    # ---- sizes: the division by the stride that used to kill the process, negative sizes, empty kernels
    _bad(name, fn + r": stride \(0\) must be at least 1", stride=0)
    _bad(name, fn + r": stride \(-1\) must be at least 1", stride=-1)
    _bad(name, fn + r": dil \(0\) must be at least 1", dil=0)
    _bad(name, fn + r": pad \(-1\) must not be negative", pad=-1)
    _bad(name, fn + r": KH \(0\) and KW \(3\) must be at least 1", KH=0)
    _bad(name, fn + r": KH \(3\) and KW \(0\) must be at least 1", KW=0)
    _bad(name, fn + r": NB \(-1\), H \(10\) and W \(12\) must not be negative", NB=-1)
    _bad(name, fn + r": NB \(0\), H \(-1\) and W \(12\) must not be negative", H=-1)
    _bad(name, fn + r": NB \(0\), H \(10\) and W \(-3\) must not be negative", W=-3)
    _bad(name, fn + r": C \(0\) must be a positive multiple of 128", C=0)
    _bad(name, fn + r": C \(-128\) must be a positive multiple of 128", C=-128)
    _bad(name, fn + r": C \(320\) must be a positive multiple of 128", C=320)
    _bad(name, fn + r": channels per deformable group \(C 512 / dgroups 8\) must be a multiple of 128", dgroups=8)
    _bad(name, fn + r": channels per deformable group \(C 512 / dgroups 0\)", dgroups=0)
    _bad(name, fn + r": channels per deformable group \(C 512 / dgroups 3\)", dgroups=3)
    _bad(name, fn + r": offset row stride off_ld \(71\) is smaller than 2\*dgroups\*KH\*KW \(72\)", off_ld=71)
    _bad(name, fn + r": offset row stride off_ld \(97\) is smaller than 2\*dgroups\*KH\*KW \(100\)", KH=5, KW=5,
         dgroups=2, off_ld=97)
    # a one-row map under a 3x3 kernel without padding has no output row: refused unless the call is empty
    # (Ho = Wo = 0 leaves a launch nothing to do, so NB = 1 is safe here too)
    _bad(name, fn + r": the output map is empty \(Ho 0, Wo 8\)", NB=1, H=1, pad=0)
    _bad(name, fn + r": the output map is empty \(Ho 6, Wo 0\)", NB=1, W=4, pad=0)
    # an empty input map under a non-empty batch is refused even where padding would give it an output map (pad = 0
    # here, so that the map check above would still stop the call if this one were missing)
    _bad(name, fn + r": H \(0\) and W \(12\) must be at least 1 when NB \(1\) > 0", NB=1, H=0, pad=0)
    _bad(name, fn + r": H \(10\) and W \(0\) must be at least 1 when NB \(2\) > 0", NB=2, W=0, pad=0)
    _bad(name, fn + r": dtype must be 0 \(fp32\) or 1 \(bf16\)", dtype=2)
    _bad(name, fn + r": dtype must be 0 \(fp32\) or 1 \(bf16\)", dtype=-1)
    # ---- pointers
    col = "col" if name == "sniper_deform_im2col" else "dcol"
    for arg in ("x", "offset", col):
        _bad(name, fn + r": x / offset / col must not be null", **{arg: 0})
    for off in (4, 8):
        _bad(name, fn + r": x must be 16-byte aligned", x=A + off)
        _bad(name, fn + r": col must be 16-byte aligned", **{col: V[1] + off})
    _bad(name, fn + r": x must be 8-byte aligned", dtype=1, x=A + 4)
    _bad(name, fn + r": col must be 8-byte aligned", dtype=1, **{col: V[1] + 2})
    _bad(name, fn + r": offset must be 4-byte aligned", offset=V[0] + 2)
    if name != "sniper_deform_im2col":
        _bad(name, fn + r": dx / doffset must not be null", dx=0)
        _bad(name, fn + r": dx / doffset must not be null", doffset=0)
        _bad(name, fn + r": doffset must be 4-byte aligned", doffset=V[3] + 2)
# the float-atomic entry adds float4 vectors into dx; the fp64-scratch entry adds single floats
for off in (4, 8):
    _bad("sniper_deform_col2im", r"deform_col2im: dx must be 16-byte aligned", dx=V[2] + off)
    _bad("sniper_deform_col2im", r"deform_col2im: dx must be 16-byte aligned", dtype=1, dx=V[2] + off)
_bad("sniper_deform_col2im_fp64acc", r"deform_col2im_fp64acc: dx must be 4-byte aligned", dx=V[2] + 2)
_bad("sniper_deform_col2im_fp64acc", r"deform_col2im_fp64acc: acc must be 8-byte aligned", acc=V[4] + 4)
_bad("sniper_deform_col2im_fp64acc", r"deform_col2im_fp64acc: acc needs", acc=0)
_bad("sniper_deform_col2im_fp64acc", r"deform_col2im_fp64acc: acc needs 0 elements, -1 given", acc_elems=-1)

for name in PS:
    _bad(name, r"psroi: num_rois \(-1\) must not be negative", num_rois=-1)
    _bad(name, r"psroi: height \(0\) and width \(\d+\) must be at least 1", height=0)
    _bad(name, r"psroi: height \(\d+\) and width \(-2\) must be at least 1", width=-2)
    _bad(name, r"psroi: rois must not be null", rois=0)
for name in ("sniper_deform_psroi_fwd", "sniper_deform_psroi_bwd", "sniper_deform_psroi_bwd_fp64acc"):
    _bad(name, r"psroi: output_dim \(0\) must be at least 1", output_dim=0, channels=0)
    _bad(name, r"psroi: group_size \(0\) must be at least 1", group_size=0, channels=0)
    _bad(name, r"psroi: pooled_size \(0\) must be at least 1", pooled_size=0)
    _bad(name, r"psroi: part_size \(-1\) must not be negative", part_size=-1)
    _bad(name, r"psroi: sample_per_part \(0\) must be at least 1", sample_per_part=0)
    _bad(name, r"psroi: channels \(255\) != output_dim\*group_size\^2 \(256\)", channels=255)
    _bad(name, r"deformable psroi: bad trans / num_classes", trans=0)
    _bad(name, r"deformable psroi: bad trans / num_classes", num_classes=3)
_bad("sniper_deform_psroi_fwd", r"psroi: layout must be 0", layout=2)
_bad("sniper_deform_psroi_bwd", r"psroi: layout must be 0", layout=-1)
for arg in ("data", "top_data"):
    _bad("sniper_deform_psroi_fwd", r"deform_psroi_fwd: data / top_data must not be null", **{arg: 0})
    _bad("sniper_psroi_fwd", r"psroi_fwd: data / top_data must not be null", **{arg: 0})
for arg in ("top_diff", "data", "data_diff"):
    _bad("sniper_deform_psroi_bwd", r"deform_psroi_bwd: top_diff / data / data_diff must not be null", **{arg: 0})
    _bad("sniper_deform_psroi_bwd_fp64acc", r"deform_psroi_bwd_fp64acc: top_diff / data / data_diff must not be null",
         **{arg: 0})
for arg in ("top_diff", "data_diff"):
    _bad("sniper_psroi_bwd", r"psroi_bwd: top_diff / data_diff must not be null", **{arg: 0})
_bad("sniper_deform_psroi_bwd", r"deformable psroi bwd: trans_diff is null", trans_diff=0)
_bad("sniper_deform_psroi_bwd_fp64acc", r"deformable psroi bwd: trans_diff is null", trans_diff=0)
_bad("sniper_psroi_fwd", r"psroi: pooled_size \(0\) must be at least 1", pooled_size=0)
_bad("sniper_psroi_bwd", r"psroi: group_size \(0\) must be at least 1", group_size=0, channels=0)
_bad("sniper_deform_psroi_bwd_fp64acc", r"deform_psroi_bwd_fp64acc: batch \(0\) must be at least 1", batch=0)
_bad("sniper_deform_psroi_bwd_fp64acc", r"deform_psroi_bwd_fp64acc: acc must be 8-byte aligned", acc=V[6] + 4)
_bad("sniper_deform_psroi_bwd_fp64acc", r"acc needs 307200 elements, 307199 given", acc_elems=2 * 20 * 30 * 256 - 1)
# shapes the NHWC kernels do not take: -2, the caller then uses sniper_deform_psroi_bwd
for change in (dict(channels=384, output_dim=384), dict(channels=256 * 9, group_size=3), dict(sample_per_part=5),
               dict(output_dim=256, num_classes=2), dict(data=A + 4), dict(top_diff=V[2] + 8), dict(data_diff=V[4] + 4)):
    _bad("sniper_deform_psroi_bwd_fp64acc", r"does not qualify for the NHWC kernels", **change)


@pytest.mark.parametrize("name,change,pattern", BAD)
def test_one_violated_rule_is_refused_by_name(name, change, pattern):
    rc, msg = _call(name, _args(name, **change))
    assert rc != 0, "%s%r was accepted" % (name, change)
    assert re.search(pattern, msg), msg


def test_fp64acc_refusal_of_a_shape_is_minus_two():
    """-2 (not -1) tells ops.deform_psroi_bwd to take the float-atomic entry instead."""
    rc, msg = _call("sniper_deform_psroi_bwd_fp64acc", _args("sniper_deform_psroi_bwd_fp64acc", sample_per_part=5))
    assert rc == -2, msg
    rc, msg = _call("sniper_deform_psroi_bwd_fp64acc", _args("sniper_deform_psroi_bwd_fp64acc", batch=0))
    assert rc == -1, msg


def test_optional_pointers_may_be_null():
    """trans / trans_diff with no_trans, top_count of the forward, sample_idx / bins: accepted."""
    for name, change in [("sniper_deform_psroi_fwd", dict(trans=0, no_trans=1)),
                         ("sniper_deform_psroi_fwd", dict(top_count=0)),
                         ("sniper_deform_psroi_bwd", dict(trans=0, trans_diff=0, no_trans=1)),
                         ("sniper_deform_psroi_bwd_fp64acc", dict(trans=0, trans_diff=0, no_trans=1)),
                         ("sniper_deform_psroi_fwd", dict(layout=0, sample_idx=V[7])),
                         ("sniper_psroi_fwd", dict(bins=V[7]))]:
        rc, msg = _call(name, _args(name, **change))
        assert rc == 0, (name, change, msg)
