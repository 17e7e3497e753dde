"""Small torch helpers shared by the three nets: pixel-major <-> channels-last views and conv wrappers.

Convolutions / plain Linear layers stay library calls (cuDNN / cuBLAS through torch, SURVEY.md §2b
"keep cuDNN initially"); everything else on the hot path goes through propainter_b200.ops.
"""
import torch
import torch.nn.functional as F

from . import autotune, config, ops


def cl(w):
    """conv weight -> channels_last memory format (done once at pack time)."""
    return w.contiguous(memory_format=torch.channels_last)


def as_nchw(pm):
    """pixel-major [n,h,w,c] (dense) -> NCHW-logical channels_last view, no copy."""
    return pm.permute(0, 3, 1, 2)


def as_pm(x):
    """NCHW-logical tensor -> pixel-major [n,h,w,c]; copies only if x is not channels_last."""
    y = x.permute(0, 2, 3, 1)
    return y if y.is_contiguous() else y.contiguous()


def pad_in_channels(w, to):
    """zero-pad a conv weight's input channels (numerically a no-op; keeps pixel rows 16-byte aligned
    and the cuDNN tensor-core path eligible)."""
    if w.shape[1] == to:
        return w
    z = w.new_zeros(w.shape[0], to - w.shape[1], *w.shape[2:])
    return torch.cat([w, z], 1)


_TORCH_ACT = {
    "none": lambda y, s: y,
    "relu": lambda y, s: F.relu_(y),
    "leaky": lambda y, s: F.leaky_relu_(y, s),
    "sigmoid": lambda y, s: torch.sigmoid_(y),
    "tanh": lambda y, s: torch.tanh_(y),
}


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def conv(x, wb, stride=1, padding=0, dilation=1, groups=1, act="none", slope=0.0, res=None, post_relu=False, out=None, pre=None):
    """conv2d + bias + activation (+ residual add, + final ReLU, + placement into a channel slice `out`).
    The conv is cuDNN; everything after it is one pass of pp_bias_act over the channels-last result (cuDNN would launch
    a separate bias add_, ATen one kernel each for the activation, the residual add and the torch.cat).  `res` / `out`
    are NCHW-logical channels_last views; `pre` (same kind of view) is added before the activation (a conv share computed
    ahead of time).  Plain conv+bias+ReLU may instead run as cuDNN's fused conv-bias-ReLU when
    that measures faster for the shape (autotune.pick; not for fp16 x, whose bias stays fp32).  Outputs whose channel
    count is not a multiple of 4 (2/3-channel heads) keep the library epilogue."""
    w, b = wb
    st, pd, dl = _pair(stride), _pair(padding), _pair(dilation)
    if not (config.FUSED_EPILOGUE and w.shape[0] % 4 == 0):
        y = F.conv2d(x, w, b, stride=st, padding=pd, dilation=dl, groups=groups)
        y = _TORCH_ACT[act](y if pre is None else y + pre, slope)
        if res is not None:
            y = y + res
        if post_relu:
            y = F.relu_(y)
        if out is not None:
            out.copy_(y)
            return out
        return y

    def own(x):
        y = F.conv2d(x, w, None, stride=st, padding=pd, dilation=dl, groups=groups)
        ypm = as_pm(y)
        o = ops.bias_act(ypm, b, act, slope, res=None if res is None else res.permute(0, 2, 3, 1), post_relu=post_relu,
                         out=None if out is None else out.permute(0, 2, 3, 1), pre=None if pre is None else pre.permute(0, 2, 3, 1))
        return as_nchw(o)

    if (act == "relu" and res is None and out is None and pre is None and not post_relu and config.AUTOTUNE
            and (b is None or x.dtype == b.dtype)):
        def fused(x):
            return torch.cudnn_convolution_relu(x, w, b, st, pd, dl, groups).contiguous(memory_format=torch.channels_last)
        return autotune.pick(("conv_relu", tuple(x.shape), tuple(w.shape), st, pd, dl, groups, x.dtype), (own, fused), x)
    return own(x)


def up2(x):
    """bilinear x2, align_corners=True, on an NCHW-logical channels_last tensor (the `deconv` blocks)."""
    if x.shape[1] % 4 == 0:
        return as_nchw(ops.upsample2x(as_pm(x)))
    return F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
