"""TEST HARNESS ONLY.  CPU stand-ins for the on-the-fly correlation ops (``ops.corr_fmap_pyramid`` /
``ops.corr_lookup_otf``), built from tests/hostsim/hostsim_otf.cpp, installed on top of tests/ops_emulation.py so the
RAFT plumbing of the on-the-fly plan (pooled levels, pair tables, plan selection) is checked against the oracle
without a GPU."""
import ctypes
import os
import subprocess

import torch

from tests import ops_emulation

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FP = ctypes.POINTER(ctypes.c_float)
IP = ctypes.POINTER(ctypes.c_int)


def build_hostsim(out_dir):
    """Compile hostsim_otf.cpp (with pp_elem.cuh) into out_dir and return the ctypes handle."""
    lib = os.path.join(out_dir, "libhostsim_otf.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", lib,
                           os.path.join(HERE, "hostsim", "hostsim_otf.cpp")])
    return ctypes.CDLL(lib)


def _fp(t):
    assert t.dtype == torch.float32 and t.is_contiguous() and not t.is_cuda
    return ctypes.cast(t.data_ptr(), FP)


def _ip(t):
    t = t.to(torch.int32).contiguous()
    return t, ctypes.cast(t.data_ptr(), IP)


def fmap_pyramid(hs, fmap, h, w):
    F_, _, D = fmap.shape
    out, src, hl, wl = [], fmap.contiguous(), h, w
    for _ in range(3):
        dst = torch.empty(F_, (hl // 2) * (wl // 2), D)
        hs.hs_fmap_pool(_fp(src), _fp(dst), ctypes.c_long(F_), hl, wl, D)
        out.append(dst)
        src, hl, wl = dst, hl // 2, wl // 2
    return out


def lookup_otf(hs, fmap, pooled, idx1, idx2, coords, out=None):
    B, h, w, _ = coords.shape
    if out is None:
        out = torch.empty(B, h, w, 324)
    i1, p1 = _ip(idx1)
    i2, p2 = _ip(idx2)
    res = torch.empty(B, h, w, 324)
    c = coords.contiguous()
    hs.hs_corr_lookup_otf(_fp(fmap.contiguous()), _fp(pooled[0]), _fp(pooled[1]), _fp(pooled[2]), fmap.shape[-1], p1, p2,
                          ctypes.c_long(B), _fp(c), _fp(res), h, w)
    out.copy_(res)
    return out


def install(monkeypatch, hostsim, hostsim_otf):
    from propainter_b200 import ops
    ops_emulation.install(monkeypatch, hostsim)
    monkeypatch.setattr(ops, "corr_fmap_pyramid", lambda fmap, h, w: fmap_pyramid(hostsim_otf, fmap, h, w))
    monkeypatch.setattr(ops, "corr_lookup_otf", lambda *a, **k: lookup_otf(hostsim_otf, *a, **k))
