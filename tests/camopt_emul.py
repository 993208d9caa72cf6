"""TEST SCAFFOLDING ONLY -- ctypes driver for the camera-pose gradient device code run by the host emulation
(tests/host_emul/emul_camopt.cpp: emul.cpp plus neurad_encode_point_mean_bwd_t and the isotropic-gaussian backward)."""
import ctypes
import os
import subprocess

import torch

from tests.host_emul import emul
from tests.host_emul.emul import _Pack, _pack_params

SO = os.path.join(emul.HERE, "libnffemul_camopt.so")
SRC = os.path.join(emul.HERE, "emul_camopt.cpp")


def build(force=False):
    deps = [SRC, emul.SRC] + [os.path.join(emul.CSRC, f) for f in ("nff_device.h", "nff_lane.h", "nff_modules.h", "nff_params.h", "simt.h")]
    if force or not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        subprocess.check_call(["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-o", SO, SRC])
    return SO
def encoding_mean_bwd(cfg, params, pdf_u, field, mean, std, times, dfeatures=None, density=None, ddensity=None, flip=None):
    """dL/d mean [N,S,3] of the module-level encoding (csrc/nff_modules.h: neurad_encode_point_mean_bwd_t; same contract as
    B200Backend.neurad_encoding_mean_bwd)."""
    lib = ctypes.CDLL(build())
    lib.emul_encoding_mean_bwd.restype = ctypes.c_int
    pk = _Pack()
    _pack_params(pk, cfg, params, pdf_u, (2, 2))
    n, s = mean.shape[0], mean.shape[1]
    ex = _Pack()
    ex.P(mean.detach().float().reshape(n, s, 3))
    ex.P(std.detach().float().reshape(n, s))
    ex.P(None if times is None else times.float().reshape(n) if times.numel() == n else times.float().reshape(n, -1)[:, 0])
    ex.P(None if flip is None else flip.float().reshape(n))
    ex.P(None if dfeatures is None else dfeatures.detach().float().reshape(n * s, dfeatures.shape[-1]))
    ex.P(None if density is None else density.detach().float().reshape(n, s))
    ex.P(None if ddensity is None else ddensity.detach().float().reshape(n, s))
    dmean = ex.P(torch.zeros(n, s, 3))
    c_ptrs, c_ints, c_floats = pk.c_arrays()
    c_extra = (ctypes.c_void_p * len(ex.ptrs))(*ex.ptrs)
    rc = lib.emul_encoding_mean_bwd(c_ptrs, c_ints, c_floats, c_extra, ctypes.c_longlong(n), ctypes.c_int(s), ctypes.c_int(field))
    assert rc == 0
    return dmean


def gaussian_bwd(bins_e, dmean):
    """Backward of `gaussian`: (d origins [N,3], d directions [N,3])."""
    lib = ctypes.CDLL(build())
    n, s = bins_e.shape[0], bins_e.shape[1] - 1
    b, dm = bins_e.float().contiguous(), dmean.detach().float().reshape(n, s, 3).contiguous()
    do, dd = torch.zeros(n, 3), torch.zeros(n, 3)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = lib.emul_gaussian_bwd(p(b), ctypes.c_longlong(n), ctypes.c_int(s), p(dm), p(do), p(dd))
    assert rc == 0
    return do, dd
