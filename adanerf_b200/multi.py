"""ctypes shim over libadanerf_b200_multi.so (include/adanerf_b200_multi.h): one process driving several GPUs of a node,
row bands + one NCCL gather per frame.  The single-device library must be loadable first (same directory)."""
import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from ._lib import AdnError, Scene, TensorDesc
from .renderer import _device_tensor, _fptr, _state_dict_of, make_scene

_HERE = os.path.dirname(os.path.abspath(__file__))
MULTI_LIB_PATH = os.environ.get("ADN_MULTI_LIB_PATH") or os.path.join(_HERE, "libadanerf_b200_multi.so")
SYMBOLS = ["adn_multi_create", "adn_multi_create_from_export_dir", "adn_multi_destroy", "adn_multi_last_error", "adn_multi_devices",
           "adn_multi_set_weights", "adn_multi_set_option", "adn_multi_band", "adn_multi_render_camera", "adn_multi_wait_frame",
           "adn_multi_last_times", "adn_multi_last_threshold", "adn_multi_last_samples"]
_multi = None


def load_multi_library():
    global _multi
    if _multi is None:
        _lib.load_library()                       # dependency: resolves libadanerf_b200.so symbols
        if not os.path.exists(MULTI_LIB_PATH):
            raise RuntimeError(f"{MULTI_LIB_PATH} is missing: run __graft_entry__.build() (needs nccl.h / libnccl)")
        lib = C.CDLL(MULTI_LIB_PATH, mode=C.RTLD_GLOBAL)
        vp, i64 = C.c_void_p, C.c_int64
        lib.adn_multi_create.argtypes = [C.POINTER(vp), C.POINTER(Scene), C.POINTER(C.c_int), C.c_int]
        lib.adn_multi_destroy.argtypes = [vp]
        lib.adn_multi_destroy.restype = None
        lib.adn_multi_last_error.argtypes = [vp]
        lib.adn_multi_last_error.restype = C.c_char_p
        lib.adn_multi_devices.argtypes = [vp]
        lib.adn_multi_set_weights.argtypes = [vp, C.c_int, C.POINTER(TensorDesc), C.c_int]
        lib.adn_multi_set_option.argtypes = [vp, C.c_char_p, i64]
        lib.adn_multi_band.argtypes = [vp, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        lib.adn_multi_band.restype = None
        lib.adn_multi_render_camera.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_float, C.c_int]
        lib.adn_multi_wait_frame.argtypes = [vp, C.POINTER(vp), vp]
        lib.adn_multi_last_times.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_float)]
        lib.adn_multi_last_threshold.argtypes = [vp, C.POINTER(C.c_float)]
        lib.adn_multi_last_samples.argtypes = [vp, C.POINTER(C.c_int64)]
        _multi = lib
    return _multi


class MultiRenderer:
    """G devices of this node, one process.  render_camera() enqueues a frame (at most two in flight), wait_frame()
    returns the oldest one as a tensor on the first device (or copies it into a host array)."""

    def __init__(self, scene, devices, sampling_net=None, shading_net=None):
        self.lib = load_multi_library()
        self.devices = [int(d) for d in devices]
        self.handle = C.c_void_p()
        sc = scene if isinstance(scene, Scene) else make_scene(**scene)
        ids = (C.c_int * len(self.devices))(*self.devices)
        st = self.lib.adn_multi_create(C.byref(self.handle), C.byref(sc), ids, len(self.devices))
        if st != 0:
            raise AdnError(st, "adn_multi_create failed")
        self._shape = [None, None]
        self._issued = self._waited = 0
        if sampling_net is not None:
            self.set_weights(0, sampling_net)
        if shading_net is not None:
            self.set_weights(1, shading_net)

    def _check(self, st):
        if st != 0:
            raise AdnError(st, (self.lib.adn_multi_last_error(self.handle) or b"").decode())

    def set_weights(self, net_id, net):
        sd = _state_dict_of(net)
        descs = (TensorDesc * len(sd))()
        keep = []
        for i, (k, v) in enumerate(sd.items()):
            v2 = v.reshape(v.shape[0], -1) if v.ndim >= 1 else v.reshape(1, 1)
            keep.append((k.encode(), v2))
            descs[i].name = keep[-1][0]
            descs[i].data = _fptr(v2)
            descs[i].rows, descs[i].cols = v2.shape[0], v2.shape[1]
        self._check(self.lib.adn_multi_set_weights(self.handle, int(net_id), descs, len(sd)))

    def set_option(self, name, value):
        """See adn_multi_set_option: "sample_budget" is the budget of the whole frame, one threshold for every band."""
        self._check(self.lib.adn_multi_set_option(self.handle, name.encode(), int(value)))

    def band(self, H, rank):
        r0, n = C.c_int(), C.c_int()
        self.lib.adn_multi_band(self.handle, int(H), int(rank), C.byref(r0), C.byref(n))
        return r0.value, n.value

    def render_camera(self, pose, rot, W, H, thr, K):
        p = np.ascontiguousarray(torch.as_tensor(pose).detach().cpu().numpy(), dtype=np.float32).reshape(3)
        r = np.ascontiguousarray(torch.as_tensor(rot).detach().cpu().numpy(), dtype=np.float32).reshape(9)
        self._check(self.lib.adn_multi_render_camera(self.handle, p.ctypes.data, r.ctypes.data, int(W), int(H), float(thr), int(K)))
        self._shape[self._issued & 1] = (int(H) * int(W), 3)
        self._issued += 1

    def wait_frame(self, host_out=None):
        """The oldest frame in flight: a [H*W, 3] fp32 view of the library's frame buffer on the first device (valid until the
        second next render_camera), or `host_out` filled when given."""
        shape = self._shape[self._waited & 1]
        ptr = C.c_void_p()
        self._check(self.lib.adn_multi_wait_frame(self.handle, C.byref(ptr), host_out.ctypes.data if host_out is not None else None))
        self._waited += 1
        if host_out is not None:
            return host_out
        return _device_tensor(ptr.value, shape, "<f4", torch.device("cuda", self.devices[0]))

    def last_times(self):
        g = len(self.devices)
        a, b = (C.c_float * g)(), (C.c_float * g)()
        self._check(self.lib.adn_multi_last_times(self.handle, a, b))
        return list(a), list(b)

    def last_threshold(self):
        """The threshold the newest frame enqueued rendered at (t* under "sample_budget").  Synchronises."""
        t = C.c_float()
        self._check(self.lib.adn_multi_last_threshold(self.handle, C.byref(t)))
        return t.value

    def last_samples(self):
        """[M of each band] of the newest frame enqueued; their sum is the frame's M.  Waits for that frame."""
        out = (C.c_int64 * len(self.devices))()
        self._check(self.lib.adn_multi_last_samples(self.handle, out))
        return list(out)

    def close(self):
        if getattr(self, "handle", None):
            self.lib.adn_multi_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
