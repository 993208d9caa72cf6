"""TEST SCAFFOLDING ONLY -- tests/fake_backend.py's CPU stand-in plus the lidar-loss operator, run by the host emulation
of its device code (tests/host_emul/emul_lidar_loss.cpp), so that NeuRADModel.get_metrics_dict / get_loss_dict run on
the CPU."""
import ctypes
import os
import subprocess
import tempfile

import torch

from tests.fake_backend import FakeBackend

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None


def emul_lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="emul_lidar_loss_"), "libemul_lidar_loss.so")
        src = os.path.join(ROOT, "tests", "host_emul", "emul_lidar_loss.cpp")
        subprocess.check_call(["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, src])
        lib = ctypes.CDLL(so)
        lib.emul_lidar_losses.restype = ctypes.c_int
        lib.emul_lidar_losses.argtypes = [ctypes.c_int64, ctypes.c_int] + [ctypes.c_void_p] * 6 + \
            [ctypes.c_int64, ctypes.c_void_p] + [ctypes.c_float] * 3 + [ctypes.c_void_p] * 3
        lib.emul_lidar_losses_bwd.restype = ctypes.c_int
        lib.emul_lidar_losses_bwd.argtypes = [ctypes.c_int64, ctypes.c_int] + [ctypes.c_void_p] * 6 + \
            [ctypes.c_int64, ctypes.c_void_p] + [ctypes.c_float] * 2 + [ctypes.c_void_p] * 7
        _LIB = lib
    return _LIB


class ObjectiveFakeBackend(FakeBackend):
    def lidar_losses(self, pred, prop, distance, did_return, intensity, gt_intensity, logits, non_return_distance,
                     non_return_mult, quantile):
        n = distance.numel()
        pr, pp, d, ret, it, gt, lg = self._lidar_loss_rows(pred, prop, distance, did_return, intensity, gt_intensity, logits)
        r = 0 if pp is None else pp.shape[0]
        out, counts, mask = torch.empty(4 + r), torch.empty(2, dtype=torch.int32), torch.empty(n, dtype=torch.bool)
        rc = emul_lib().emul_lidar_losses(n, r, pr.data_ptr(), None if pp is None else pp.data_ptr(), d.data_ptr(),
                                          ret.data_ptr(), it.data_ptr(), gt.data_ptr(), gt.stride(0), lg.data_ptr(),
                                          non_return_distance, non_return_mult, quantile, out.data_ptr(), mask.data_ptr(),
                                          counts.data_ptr())
        assert rc == 0
        return out, counts, mask

    def lidar_losses_bwd(self, pred, prop, distance, did_return, intensity, gt_intensity, logits, non_return_distance,
                         non_return_mult, mask, counts, grad_out):
        n = distance.numel()
        pr, pp, d, ret, it, gt, lg = self._lidar_loss_rows(pred, prop, distance, did_return, intensity, gt_intensity, logits)
        r = 0 if pp is None else pp.shape[0]
        d_pred, d_int, d_lg, d_prop = torch.empty(n), torch.empty(n), torch.empty(n), torch.empty(r, n)
        g = grad_out.detach().float().contiguous()
        rc = emul_lib().emul_lidar_losses_bwd(n, r, pr.data_ptr(), None if pp is None else pp.data_ptr(), d.data_ptr(),
                                              ret.data_ptr(), it.data_ptr(), gt.data_ptr(), gt.stride(0), lg.data_ptr(),
                                              non_return_distance, non_return_mult, mask.data_ptr(), counts.data_ptr(),
                                              g.data_ptr(), d_pred.data_ptr(), d_prop.data_ptr(), d_int.data_ptr(),
                                              d_lg.data_ptr())
        assert rc == 0
        return d_pred, d_prop, d_int, d_lg
