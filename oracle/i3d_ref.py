"""Oracle (test infrastructure): InceptionI3d.extract_features (core/metrics.py:195-569) restated functionally in plain
fp32 torch over a state_dict, on whatever device its tensors are.  Unlike the product it keeps the reference's NCDHW
layout, pads with F.pad, applies eval batch-norm unfolded and concatenates the Inception branches; it shares no code
with propainter_b200.model.i3d.

    feats = extract_features(sd, x)                               # x [B,3,T,H,W] float32 in [0, 1] -> [B,1024]
    feats, maps = extract_features(sd, x, return_maps=True)       # + every endpoint's map
"""
import torch
import torch.nn.functional as F

ENDPOINTS = ('Conv3d_1a_7x7', 'MaxPool3d_2a_3x3', 'Conv3d_2b_1x1', 'Conv3d_2c_3x3', 'MaxPool3d_3a_3x3', 'Mixed_3b',
             'Mixed_3c', 'MaxPool3d_4a_3x3', 'Mixed_4b', 'Mixed_4c', 'Mixed_4d', 'Mixed_4e', 'Mixed_4f',
             'MaxPool3d_5a_2x2', 'Mixed_5b', 'Mixed_5c')
POOLS = {'MaxPool3d_2a_3x3': ((1, 3, 3), (1, 2, 2)), 'MaxPool3d_3a_3x3': ((1, 3, 3), (1, 2, 2)),   # :420-421, :444-445
         'MaxPool3d_4a_3x3': ((3, 3, 3), (2, 2, 2)), 'MaxPool3d_5a_2x2': ((2, 2, 2), (2, 2, 2))}   # :463-464, :500-501


def compute_pad(k, s, n):
    """Unit3D.compute_pad / MaxPool3dSamePadding.compute_pad (core/metrics.py:196-200, :258-262)"""
    if n % s == 0:
        return max(k - s, 0)
    return max(k - (n % s), 0)


def same_pad(x, kernel, stride):
    """the F.pad of Unit3D.forward / MaxPool3dSamePadding.forward (core/metrics.py:204-217, :266-279)"""
    pad = []
    for d in (2, 1, 0):                                              # F.pad order: W, H, T
        p = compute_pad(kernel[d], stride[d], x.shape[2 + d])
        pad += [p // 2, p - p // 2]
    return F.pad(x, pad)


def unit3d(sd, p, x, kernel, stride=(1, 1, 1)):
    """Unit3D.forward (core/metrics.py:264-286): 'same' F.pad, conv3d (padding 0, no bias), eval BatchNorm3d(eps=1e-3),
    ReLU"""
    x = F.conv3d(same_pad(x, kernel, stride), sd[p + ".conv3d.weight"], None, stride)
    x = F.batch_norm(x, sd[p + ".bn.running_mean"], sd[p + ".bn.running_var"], sd[p + ".bn.weight"], sd[p + ".bn.bias"],
                     False, 0.01, 1e-3)
    return F.relu(x)


def maxpool_same(x, kernel, stride):
    """MaxPool3dSamePadding.forward (core/metrics.py:202-218): zero F.pad, then nn.MaxPool3d(kernel, stride, padding=0)"""
    return F.max_pool3d(same_pad(x, kernel, stride), kernel, stride)


def inception(sd, p, x):
    """InceptionModule.forward (core/metrics.py:326-331)"""
    b0 = unit3d(sd, p + ".b0", x, (1, 1, 1))
    b1 = unit3d(sd, p + ".b1b", unit3d(sd, p + ".b1a", x, (1, 1, 1)), (3, 3, 3))
    b2 = unit3d(sd, p + ".b2b", unit3d(sd, p + ".b2a", x, (1, 1, 1)), (3, 3, 3))
    b3 = unit3d(sd, p + ".b3b", maxpool_same(x, (3, 3, 3), (1, 1, 1)), (1, 1, 1))
    return torch.cat([b0, b1, b2, b3], dim=1)


def endpoint(sd, name, x):
    if name == 'Conv3d_1a_7x7':
        return unit3d(sd, name, x, (7, 7, 7), (2, 2, 2))                                     # :409-415
    if name == 'Conv3d_2b_1x1':
        return unit3d(sd, name, x, (1, 1, 1))                                                # :426-430
    if name == 'Conv3d_2c_3x3':
        return unit3d(sd, name, x, (3, 3, 3))                  # :435-439 (its padding=1 argument is unused, :249)
    if name in POOLS:
        return maxpool_same(x, *POOLS[name])
    return inception(sd, name, x)                                                            # :449-517


@torch.no_grad()
def extract_features(sd, x, target_endpoint='Logits', return_maps=False):
    """InceptionI3d.extract_features (core/metrics.py:560-569) for final_endpoint='Logits'"""
    maps = {}
    for name in ENDPOINTS:
        x = endpoint(sd, name, x)
        maps[name] = x
        if name == target_endpoint:
            break
    out = x.mean(4).mean(3).mean(2) if target_endpoint == 'Logits' else x
    return (out, maps) if return_maps else out


def video_from_u8(frames_u8):
    """to_tensors (core/utils.py:151-170) of a uint8 video [T,H,W,3] (numpy or tensor) + unsqueeze(0) + transpose(1, 2)
    (core/metrics.py:75,183) -> [1,3,T,H,W] float32 in [0, 1]"""
    u8 = torch.as_tensor(frames_u8)
    return u8.permute(3, 0, 1, 2).float().div(255)[None].contiguous()
