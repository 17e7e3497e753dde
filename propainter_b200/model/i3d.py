"""The I3D feature network behind VFID on the H100 path.

Drop-in for the reference's ``InceptionI3d`` (core/metrics.py:334-569) as the evaluation uses it (init_i3d_model,
get_i3d_activations, core/metrics.py:62-82,153-188): same constructor, same state_dict (pytorch-i3d's
``i3d_rgb_imagenet.pt`` loads ``strict=True``), same ``extract_features(x, target_endpoint)`` results.
What differs is the execution plan:
  * feature maps live pixel-major (NDHWC); the 57 convolutions are cuDNN conv3d on channels_last_3d tensors with
    eval BatchNorm folded into the weights once per device
  * the input conversion and Conv3d_1a_7x7's asymmetric 'same' border are one kernel (``ops.i3d_input``), so that conv
    runs unpadded and the F.pad copy disappears; the other 'same' conv borders are symmetric and are cuDNN padding
  * BN shift + ReLU and the placement of each Inception branch into its slice of the block output are one
    ``ops.bias_act`` pass (no torch.cat); the three 1x1x1 heads that read a block's input (b0, b1a, b2a) are one conv
  * MaxPool3dSamePadding and the final mean over (T, H, W) are ``ops.maxpool3d_same`` / ``ops.mean_thw``
Only ``final_endpoint='Logits'`` (what every reference caller builds) is supported, and the Kinetics classifier
``forward`` is not: no metric uses it.  Its parameters stay in the state_dict so checkpoints load.
"""
import torch
import torch.nn.functional as F

from .. import ops
from .._params import ParamNet
from ..schemas import I3D_INCEPTION, i3d_schema

VALID_ENDPOINTS = (
    'Conv3d_1a_7x7', 'MaxPool3d_2a_3x3', 'Conv3d_2b_1x1', 'Conv3d_2c_3x3', 'MaxPool3d_3a_3x3', 'Mixed_3b', 'Mixed_3c',
    'MaxPool3d_4a_3x3', 'Mixed_4b', 'Mixed_4c', 'Mixed_4d', 'Mixed_4e', 'Mixed_4f', 'MaxPool3d_5a_2x2', 'Mixed_5b',
    'Mixed_5c', 'Logits', 'Predictions',
)
# the pooling endpoints: (kernel, stride), core/metrics.py:420-421,444-445,463-464,500-501
_POOLS = {
    'MaxPool3d_2a_3x3': ((1, 3, 3), (1, 2, 2)),
    'MaxPool3d_3a_3x3': ((1, 3, 3), (1, 2, 2)),
    'MaxPool3d_4a_3x3': ((3, 3, 3), (2, 2, 2)),
    'MaxPool3d_5a_2x2': ((2, 2, 2), (2, 2, 2)),
}
_BN_EPS = 1e-3                                          # Unit3D's BatchNorm3d(eps=0.001), core/metrics.py:254-256


def _pm5(y):
    """NCDHW-logical conv output -> pixel-major [B,T,H,W,C]; no copy when cuDNN returned channels_last_3d"""
    p = y.permute(0, 2, 3, 4, 1)
    return p if p.is_contiguous() else p.contiguous()


def _ncdhw(pm):
    """pixel-major [B,T,H,W,C] -> NCDHW-logical channels_last_3d view, no copy"""
    return pm.permute(0, 4, 1, 2, 3)


class InceptionI3d(ParamNet):
    VALID_ENDPOINTS = VALID_ENDPOINTS

    def __init__(self, num_classes=400, spatial_squeeze=True, final_endpoint='Logits', name='inception_i3d', in_channels=3,
                 dropout_keep_prob=0.5, seed=None):
        if final_endpoint not in VALID_ENDPOINTS:
            raise ValueError('Unknown final endpoint %s' % final_endpoint)
        if final_endpoint != 'Logits':
            raise ValueError(f"final_endpoint={final_endpoint!r}: only 'Logits' (the full feature network every VFID caller "
                             "builds) is supported")
        if in_channels != 3:
            raise ValueError(f"in_channels={in_channels}: the input kernel packs RGB videos (3 channels)")
        super().__init__(i3d_schema(num_classes, in_channels), seed=seed)
        self._num_classes = num_classes
        self._spatial_squeeze = spatial_squeeze
        self._final_endpoint = final_endpoint
        self.name = name

    def load_state_dict(self, state_dict, strict=True, assign=False):
        """As nn.Module's.  A checkpoint without `num_batches_tracked` buffers (written before they existed, as
        pytorch-i3d's were) gets them as 0, the rule BatchNorm3d applies to such state dicts; they are not used in eval."""
        sd = dict(state_dict)
        for k in self._keys:
            if k.endswith(".bn.num_batches_tracked") and k not in sd and k[:-len("num_batches_tracked")] + "running_mean" in sd:
                sd[k] = torch.zeros((), dtype=torch.long)
        return super().load_state_dict(sd, strict=strict, assign=assign)

    def forward(self, x):
        raise NotImplementedError("InceptionI3d.forward (the Kinetics classifier: avg_pool + logits) is not implemented; "
                                  "VFID uses extract_features")

    # ------------------------------------------------------------------ weights
    def _folded(self, key):
        """Unit3D `key` with its eval BatchNorm folded: (weight * scale [Cout,Cin,kt,kh,kw], shift [Cout]), scale =
        gamma / sqrt(var + eps) and shift = beta - mean * scale in fp32."""
        P = self.P
        s = P[key + ".bn.weight"] / torch.sqrt(P[key + ".bn.running_var"] + _BN_EPS)
        return P[key + ".conv3d.weight"] * s.view(-1, 1, 1, 1, 1), (P[key + ".bn.bias"] - P[key + ".bn.running_mean"] * s)

    def _unit(self, key):
        def build():
            w, b = self._folded(key)
            if key == "Conv3d_1a_7x7":                      # the zero 4th input channel of ops.i3d_input
                w = torch.cat([w, w.new_zeros(w.shape[0], 1, *w.shape[2:])], 1)
            return w.contiguous(memory_format=torch.channels_last_3d), b.contiguous()
        return self.packed("unit:" + key, build)

    def _heads(self, name):
        """b0 | b1a | b2a of an Inception block as one 1x1x1 conv (concatenated output channels)"""
        def build():
            ws, bs = zip(*[self._folded(f"{name}.{h}") for h in ("b0", "b1a", "b2a")])
            return torch.cat(ws, 0).contiguous(memory_format=torch.channels_last_3d), torch.cat(bs).contiguous()
        return self.packed("heads:" + name, build)

    # ------------------------------------------------------------------ layers
    def _conv(self, x, key, stride=1, padding=0, out=None):
        """Unit3D.forward: conv3d (cuDNN) + folded BN + ReLU (pp_bias_act, into `out` when given)"""
        w, b = self._unit(key)
        y = _pm5(F.conv3d(_ncdhw(x), w, None, stride, padding))
        return ops.bias_act(y, b, "relu", out=out)

    def _inception(self, x, name, cout):
        """InceptionModule.forward (core/metrics.py:326-331): every branch's epilogue writes its slice of the output"""
        c0, c1a, c1b, c2a, c2b, c3b = cout
        B, T, H, W, _ = x.shape
        out = torch.empty(B, T, H, W, c0 + c1b + c2b + c3b, device=x.device, dtype=torch.float32)
        wh, bh = self._heads(name)
        y = _pm5(F.conv3d(_ncdhw(x), wh, None))
        ops.bias_act(y[..., :c0], bh[:c0], "relu", out=out[..., :c0])
        t1 = ops.bias_act(y[..., c0:c0 + c1a], bh[c0:c0 + c1a], "relu", out=torch.empty(B, T, H, W, c1a, device=x.device))
        t2 = ops.bias_act(y[..., c0 + c1a:], bh[c0 + c1a:], "relu", out=torch.empty(B, T, H, W, c2a, device=x.device))
        self._conv(t1, name + ".b1b", padding=1, out=out[..., c0:c0 + c1b])     # 'same' for k = 3, s = 1 is 1 / 1
        self._conv(t2, name + ".b2b", padding=1, out=out[..., c0 + c1b:c0 + c1b + c2b])
        self._conv(ops.maxpool3d_same(x, (3, 3, 3), (1, 1, 1)), name + ".b3b", out=out[..., c0 + c1b + c2b:])
        return out

    def _endpoint(self, ep, x):
        if ep == 'Conv3d_1a_7x7':
            return self._conv(ops.i3d_input(x), ep, stride=2)
        if ep in _POOLS:
            return ops.maxpool3d_same(x, *_POOLS[ep])
        if ep == 'Conv3d_2b_1x1':
            return self._conv(x, ep)
        if ep == 'Conv3d_2c_3x3':
            return self._conv(x, ep, padding=1)
        return self._inception(x, ep, _INCEPTION_OUT[ep])

    @torch.no_grad()
    def _features(self, video, target_endpoint):
        """the endpoint loop of extract_features (core/metrics.py:560-569) over ops.i3d_input's source `video`"""
        x = video
        for ep in VALID_ENDPOINTS[:16]:                     # the built endpoints, Conv3d_1a_7x7 .. Mixed_5c
            x = self._endpoint(ep, x)
            if ep == target_endpoint:
                break
        if target_endpoint == 'Logits':
            return ops.mean_thw(x)
        return x.permute(0, 4, 1, 2, 3).contiguous()

    def extract_features(self, x, target_endpoint='Logits'):
        """x [B,3,T,H,W] float32 in [0, 1] on the device (get_i3d_activations' transpose(1, 2) of the to_tensors video).
        'Logits' -> [B,1024], the mean over (T, H, W) of Mixed_5c; an endpoint name -> that endpoint's map [B,C,T,H,W];
        any other name runs the whole network and returns Mixed_5c's map, as the reference's loop does."""
        if x.dim() != 5 or x.shape[1] != 3:
            raise ValueError(f"extract_features: expected [B,3,T,H,W], got {tuple(x.shape)}")
        return self._features(x.contiguous(), target_endpoint)

    def features_u8(self, frames_u8):
        """uint8 frames [B,T,H,W,3] on the device -> [B,1024]: get_i3d_activations of the to_tensors videos, with the
        uint8 -> [0, 1] conversion fused into the input kernel."""
        if frames_u8.dim() != 5 or frames_u8.shape[-1] != 3:
            raise ValueError(f"features_u8: expected uint8 [B,T,H,W,3], got {tuple(frames_u8.shape)}")
        return self._features(frames_u8, 'Logits')


_INCEPTION_OUT = {name: cout for name, _, cout in I3D_INCEPTION}
