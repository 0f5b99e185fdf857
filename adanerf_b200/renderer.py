"""Python host side of the H100 renderer: mirrors the call surface of the reference's
`TrainConfig.inference` (src/train_data.py:278-299) as `render(rays, sampling_net, shading_net,
adaptiveSamplingThreshold)` on top of the C ABI.  PyTorch is used only for device memory and streams."""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import AdnError, AuxOutputs, Scene, Stats, TensorDesc


def enc_columns(n_bands):
    """Columns of one encoded 3-vector with n_bands frequency bands (3 + 6 n_bands); a negative count is posEnc none,
    the 3-column identity."""
    return 3 + 6 * max(0, int(n_bands))


def scene_columns(sc):
    """(sampling-net inputs, shading-net position columns, shading-net view columns) of a Scene, as adn_create reads its
    band counts: a negative one is posEnc none; the sampling net's 0 is "the shading net's"."""
    p0 = sc.n_freq_pos0 if sc.n_freq_pos0 else sc.n_freq_pos
    d0 = sc.n_freq_dir0 if sc.n_freq_dir0 else sc.n_freq_dir
    return enc_columns(p0) + enc_columns(d0), enc_columns(sc.n_freq_pos), enc_columns(sc.n_freq_dir)


def make_scene(view_cell_center, view_cell_size, depth_range, max_depth, fov, z_near=0.001, z_far=1.0,
               n_freq_pos=10, n_freq_dir=4, use_ndc=False, w=0, h=0, focal=0.0, n_freq_pos0=None, n_freq_dir0=None, **_):
    """use_ndc: the NDC / LLFF variant (configs/fine_training_ndc.ini); w, h, focal = the dataset's image size and focal
    length that ndc_rays uses (src/features.py:350-351,430); the sampling net then takes the "2-2" encoding (30 features)
    unless n_freq_pos0 / n_freq_dir0 say otherwise.
    n_freq_pos / n_freq_dir: the shading net's posEncArgs band counts (-1: posEnc none); n_freq_pos0 / n_freq_dir0 the
    sampling net's (0: the same as the shading net's; -1: posEnc none or zero bands)."""
    s = Scene()
    s.view_cell_center[:] = [float(x) for x in view_cell_center]
    s.view_cell_size[:] = [float(x) for x in view_cell_size]
    s.depth_range[:] = [float(x) for x in depth_range]
    s.max_depth, s.fov, s.z_near, s.z_far = float(max_depth), float(fov), float(z_near), float(z_far)
    s.n_freq_pos, s.n_freq_dir = int(n_freq_pos), int(n_freq_dir)
    s.use_ndc, s.ndc_w, s.ndc_h, s.ndc_focal = int(bool(use_ndc)), int(w or 0), int(h or 0), float(focal or 0.0)
    s.n_freq_pos0 = int(n_freq_pos0) if n_freq_pos0 is not None else (2 if use_ndc else 0)
    s.n_freq_dir0 = int(n_freq_dir0) if n_freq_dir0 is not None else (2 if use_ndc else 0)
    return s


# the observer src/evaluate.py:123-126 evaluates FLIP for: 0.7 m from a 0.7 m wide 3840-pixel screen, in pixels per degree
EVALUATE_PPD = 0.7 * (3840 / 0.7) * (np.pi / 180)

# adn_image_iwssim's layouts (ADN_IWSSIM_EVALUATE_RGB, ADN_IWSSIM_GRAY) and its smallest frame side
IWSSIM_LAYOUTS = {"gray": 0, "evaluate": 1}
IWSSIM_MIN_SIZE = 161


def _fptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _state_dict_of(net):
    if hasattr(net, "state_dict"):
        net = net.state_dict()
    return {k: np.ascontiguousarray(v.detach().cpu().float().numpy() if isinstance(v, torch.Tensor) else np.asarray(v, np.float32))
            for k, v in net.items()}


class Renderer:
    """One context per device.  `sampling_net` / `shading_net`: nn.Module or state_dict with the
    reference's parameter names (src/models.py:71-76, :226-244).  A plain NeRF (rayMarchSampler LinearlySpacedZNearZFar) has
    no sampling net: pass its network as shading_net and set option "sampler" to 2."""

    def __init__(self, scene, device=0, sampling_net=None, shading_net=None, _handle=None):
        self.lib = _lib.load_library()
        self.device = int(device)
        self.handle = C.c_void_p()
        self._registered = {}    # address -> numpy array page-locked through register_host_buffer (kept alive here)
        self._reduce_cb = None    # the budget group's ctypes callback (set_budget_group), kept alive while installed
        self._reduce_error = None  # the exception the reducer raised in the failing call
        self.n_feat0 = 90        # sampling-net input features (30 with the "2-2" encoding of the NDC configs)
        self.n_feat1 = 90        # shading-net input features: position, then view columns
        if _handle is not None:
            self.handle = _handle
        else:
            sc = scene if isinstance(scene, Scene) else make_scene(**scene)
            self._check(self.lib.adn_create(C.byref(self.handle), C.byref(sc), self.device), create=True)
            self._set_columns(sc)
        if sampling_net is not None:
            self.set_weights(0, sampling_net)
        if shading_net is not None:
            self.set_weights(1, shading_net)

    @classmethod
    def from_export_dir(cls, path, device=0):
        """Loads the reference's export directory (src/export.py:28-93). Returns (renderer, thr, K).  A FromClassifiedDepth
        export comes back with options "sampler" = 1 and its "pdf_transform" set (export_sampler reads them from
        config.ini); its thr is not used.  A one-network LinearlySpacedZNearZFar export comes back with its net in the
        shading slot and option "sampler" = 2."""
        lib = _lib.load_library()
        h, thr, k = C.c_void_p(), C.c_float(), C.c_int()
        st = lib.adn_create_from_export_dir(C.byref(h), str(path).encode(), int(device), C.byref(thr), C.byref(k))
        if st != 0:
            raise AdnError(st, f"loading export dir {path}")
        r = cls(None, device=device, _handle=h)
        sc, nt = Scene(), (C.c_int * 2)()
        if lib.adn_probe_export_dir(str(path).encode(), C.byref(sc), None, None, nt) == 0:
            r._set_columns(sc)
        return r, float(thr.value), int(k.value)

    def _set_columns(self, sc):
        n0, n_p, n_v = scene_columns(sc)
        self.n_feat0, self.n_feat1 = n0, n_p + n_v

    def _check(self, st, create=False):
        if st != 0:
            detail = "" if create or not self.handle else (self.lib.adn_last_error(self.handle) or b"").decode()
            cause, self._reduce_error = self._reduce_error, None
            raise AdnError(st, detail) from cause

    def close(self):
        if getattr(self, "handle", None):
            self.lib.adn_destroy(self.handle)      # also ends every host-buffer registration
            self.handle = None
            self._registered = {}

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- weights / options ---------------------------------------------------------------
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
        self._check(self.lib.adn_set_weights(self.handle, int(net_id), descs, len(sd)))

    def set_option(self, name, value):
        self._check(self.lib.adn_set_option(self.handle, name.encode(), int(value)))

    def set_budget_group(self, fn):
        """Joins a budget group (adn_set_budget_group): budgeted calls on this renderer and on the other members choose one
        threshold under one budget, as one renderer would over all their rays.  fn(words) must sum `words` -- an int64
        tensor on this renderer's device aliasing the library's uint64 histogram words -- in place across all members, on
        the current stream (the call's), e.g. lambda t: dist.all_reduce(t, group=g).  The counts stay below 2^63, so the
        signed sum is the unsigned one.  It runs on the thread that makes the call, once per select round.  An exception
        in fn fails that call (AdnError, raised from the exception).  fn = None leaves the group."""
        if fn is None:
            self._check(self.lib.adn_set_budget_group(self.handle, _lib.BUDGET_REDUCE_FN(), None))
            self._reduce_cb = None
            return
        dev = self._dev()

        def reduce(_user, words, n_words, stream):
            try:
                t = _device_tensor(words, (n_words,), "<i8", dev)
                st = torch.cuda.ExternalStream(stream, device=dev) if stream else torch.cuda.default_stream(dev)
                with torch.cuda.device(dev), torch.cuda.stream(st):
                    fn(t)
                return 0
            except BaseException as e:     # the library sees a failed reduction; _check raises from e
                self._reduce_error = e
                return 1

        cb = _lib.BUDGET_REDUCE_FN(reduce)
        self._check(self.lib.adn_set_budget_group(self.handle, cb, None))
        self._reduce_cb = cb               # the library calls it until the group is left

    def net_dims(self, net_id):
        n_in, n_out = C.c_int(), C.c_int()
        self._check(self.lib.adn_net_dims(self.handle, int(net_id), C.byref(n_in), C.byref(n_out)))
        return n_in.value, n_out.value

    def depth_cells(self):
        """D, the depth cells the sampling net classifies (multiDepthFeatures: 32, 64, 128 or 256): its output width, the
        row width of raw0 / oracle_weights.  128 while no sampling net is set."""
        try:
            return self.net_dims(0)[1]
        except AdnError:
            return 128

    def net_shape(self, net_id):
        """(depth, width, skip) the library inferred from the weights of network net_id; skip = -1 when it has none."""
        d, w, s = C.c_int(), C.c_int(), C.c_int()
        self._check(self.lib.adn_net_shape(self.handle, int(net_id), C.byref(d), C.byref(w), C.byref(s)))
        return d.value, w.value, s.value

    def register_host_buffer(self, array):
        """Page-locks a numpy array in place so render_rays_host / render_camera_host DMA straight from / to it.  The
        renderer keeps a reference (the memory must outlive the registration); unregister_host_buffer or close() ends it."""
        if not (isinstance(array, np.ndarray) and array.flags["C_CONTIGUOUS"]):
            raise ValueError("register_host_buffer: need a C-contiguous numpy array")
        self._check(self.lib.adn_register_host_buffer(self.handle, array.ctypes.data, array.nbytes))
        self._registered[array.ctypes.data] = array

    def unregister_host_buffer(self, array):
        self._check(self.lib.adn_unregister_host_buffer(self.handle, array.ctypes.data))
        self._registered.pop(array.ctypes.data, None)

    def stats(self):
        s = Stats()
        self._check(self.lib.adn_get_stats(self.handle, C.byref(s)))
        return dict(n_rays=s.n_rays, n_samples=s.n_samples, ms_stage=list(s.ms_stage), kernel_launches=s.kernel_launches)

    def last_threshold(self):
        """The threshold the last render used: the one chosen under set_option("sample_budget", B), else the `thr` it was
        given.  Synchronises."""
        t = C.c_float()
        self._check(self.lib.adn_last_threshold(self.handle, C.byref(t)))
        return t.value

    # ---- helpers -------------------------------------------------------------------------
    def _dev(self):
        return torch.device("cuda", self.device)

    @staticmethod
    def _pose_rot(pose, rot):
        p = np.ascontiguousarray(np.asarray(pose.detach().cpu() if isinstance(pose, torch.Tensor) else pose, dtype=np.float32).reshape(3))
        r = np.ascontiguousarray(np.asarray(rot.detach().cpu() if isinstance(rot, torch.Tensor) else rot, dtype=np.float32).reshape(9))
        return p, r

    @staticmethod
    def _stream():
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def _f32(self, t):
        t = t.to(device=self._dev(), dtype=torch.float32)
        return t if t.is_contiguous() else t.contiguous()

    # ---- the hot path --------------------------------------------------------------------
    AUX_KEYS = ("weights", "alpha", "z_vals", "depth_map", "acc_map", "disp_map", "depth_est")

    def render_rays(self, pose, rot, dirs, thr, K, want_nsamples=True, want_oracle_weights=False, want_aux=False, out=None,
                    aux_out=None):
        """dirs [N,3] (cuda tensor) -> dict(rgb [N,3], n_samples [N] int32, oracle_weights [N,D]; D = depth_cells()).
        want_aux: True or an iterable of AUX_KEYS -> additionally weights / alpha / z_vals [N,K] and depth_map /
        acc_map / disp_map / depth_est [N] (adaptive_raw2outputs' other outputs, src/nerf_raymarch_common.py:137-144;
        depth_est = "NeRFOutputDepth", src/features.py:574-577).  aux_out: dict of contiguous float32 tensors on the
        renderer's device to write requested aux outputs into instead of new ones."""
        p, r = self._pose_rot(pose, rot)
        d = self._f32(dirs).reshape(-1, 3)
        n = d.shape[0]
        out, aux = self._ray_outputs("render_rays", n, K, want_nsamples, want_oracle_weights, want_aux, out, aux_out)
        ptr = lambda t: t.data_ptr() if t is not None else None
        with torch.cuda.device(self.device):
            self._check(self.lib.adn_render_rays_aux(self.handle, _fptr(p), _fptr(r), d.data_ptr(), n, float(thr), int(K),
                                                     out["rgb"].data_ptr(), ptr(out["n_samples"]), ptr(out["oracle_weights"]),
                                                     C.byref(aux) if aux is not None else None, self._stream()))
        return out

    def _ray_outputs(self, who, n, K, want_nsamples, want_oracle_weights, want_aux, out, aux_out):
        """The output tensors of a render over n rays (render_rays, render_views) and the adn_aux_outputs that point at the
        requested aux ones (None when none is)."""
        if out is not None and (out.dtype != torch.float32 or out.numel() != 3 * n or not out.is_contiguous() or out.device != self._dev()):
            raise ValueError(f"{who}: out must be a contiguous float32 [N,3] tensor on the renderer's device")
        rgb = out if out is not None else torch.empty((n, 3), dtype=torch.float32, device=self._dev())
        ns = torch.empty((n,), dtype=torch.int32, device=self._dev()) if want_nsamples else None
        ow = torch.empty((n, self.depth_cells()), dtype=torch.float32, device=self._dev()) if want_oracle_weights else None
        out = dict(rgb=rgb, n_samples=ns, oracle_weights=ow)
        aux = None
        if want_aux:
            aux = AuxOutputs()
            for k in self.AUX_KEYS if want_aux is True else tuple(want_aux):
                if k not in self.AUX_KEYS:
                    raise KeyError(f"unknown auxiliary output {k!r}")
                shape = (n, int(K)) if k in ("weights", "alpha", "z_vals") else (n,)
                t = (aux_out or {}).get(k)
                if t is None:
                    t = torch.empty(shape, dtype=torch.float32, device=self._dev())
                elif t.dtype != torch.float32 or tuple(t.shape) != shape or not t.is_contiguous() or t.device != self._dev():
                    raise ValueError(f"{who}: aux_out[{k!r}] must be a contiguous float32 {list(shape)} tensor on the renderer's device")
                out[k] = t
                setattr(aux, "d_" + k, t.data_ptr())
        return out, aux

    @staticmethod
    def _view_tables(poses, rots):
        """poses [V,3] and rots [V,3,3] (tensors or arrays) -> contiguous float32 host arrays [V,3], [V,9] and V."""
        host = lambda x: np.asarray(x.detach().cpu() if isinstance(x, torch.Tensor) else x, dtype=np.float32)
        p, r = host(poses), host(rots)
        v = p.reshape(-1, 3).shape[0] if p.size % 3 == 0 else -1
        if p.size != 3 * v or r.size != 9 * v or v < 1:
            raise ValueError(f"views: poses must be [V,3] and rots [V,3,3] for the same V >= 1, got {p.shape} and {r.shape}")
        return np.ascontiguousarray(p.reshape(v, 3)), np.ascontiguousarray(r.reshape(v, 9)), v

    def render_views(self, poses, rots, dirs, thr, K, want_nsamples=True, want_oracle_weights=False, want_aux=False, out=None,
                     aux_out=None):
        """V cameras in one call (adn_render_views_rays): poses [V,3], rots [V,3,3], dirs [V,N,3] (cuda tensor) -> the dict
        of render_rays over the V N rays, view-major ([V N, ...]: ray v N + i is ray i of view v).  Without a sample budget
        this is bit for bit the V render_rays calls concatenated; under one, one threshold covers all views."""
        p, r, v = self._view_tables(poses, rots)
        d = self._f32(dirs).reshape(-1, 3)
        if d.shape[0] % v:
            raise ValueError(f"render_views: dirs must be [V,N,3] with V = {v}, got {tuple(dirs.shape)}")
        n = d.shape[0]
        out, aux = self._ray_outputs("render_views", n, K, want_nsamples, want_oracle_weights, want_aux, out, aux_out)
        ptr = lambda t: t.data_ptr() if t is not None else None
        with torch.cuda.device(self.device):
            self._check(self.lib.adn_render_views_rays(self.handle, v, _fptr(p), _fptr(r), d.data_ptr(), n // v, float(thr), int(K),
                                                       out["rgb"].data_ptr(), ptr(out["n_samples"]), ptr(out["oracle_weights"]),
                                                       C.byref(aux) if aux is not None else None, self._stream()))
        return out

    def render_views_camera(self, poses, rots, W, H, thr, K, rgba8=False, want_nsamples=False):
        """V whole W x H frames in one call (adn_render_views_camera / _rgba8) -> dict(rgb [V*H*W, 3] float32, n_samples
        [V*H*W] int32 or None), or with rgba8=True the viewer's pixels [V*H*W, 4] uint8."""
        p, r, v = self._view_tables(poses, rots)
        n = v * int(W) * int(H)
        dev = self._dev()
        with torch.cuda.device(self.device):
            if rgba8:
                px = torch.empty((n, 4), dtype=torch.uint8, device=dev)
                self._check(self.lib.adn_render_views_camera_rgba8(self.handle, v, _fptr(p), _fptr(r), int(W), int(H), float(thr),
                                                                   int(K), px.data_ptr(), self._stream()))
                return px
            rgb = torch.empty((n, 3), dtype=torch.float32, device=dev)
            ns = torch.empty((n,), dtype=torch.int32, device=dev) if want_nsamples else None
            self._check(self.lib.adn_render_views_camera(self.handle, v, _fptr(p), _fptr(r), int(W), int(H), float(thr), int(K),
                                                         rgb.data_ptr(), ns.data_ptr() if ns is not None else None, self._stream()))
        return dict(rgb=rgb, n_samples=ns)

    def render_camera(self, pose, rot, W, H, thr, K, row0=0, rows=None, out=None, want_nsamples=False):
        """Renders image rows [row0, row0+rows) of a WxH pinhole frame; rays generated on the device."""
        rows = H - row0 if rows is None else rows
        p, r = self._pose_rot(pose, rot)
        n = rows * W
        rgb = out if out is not None else torch.empty((n, 3), dtype=torch.float32, device=self._dev())
        ns = torch.empty((n,), dtype=torch.int32, device=self._dev()) if want_nsamples else None
        with torch.cuda.device(self.device):
            self._check(self.lib.adn_render_camera(self.handle, _fptr(p), _fptr(r), W, H, row0, rows, float(thr), int(K),
                                                   rgb.data_ptr(), ns.data_ptr() if ns is not None else None, self._stream()))
        return dict(rgb=rgb, n_samples=ns)

    def render_camera_rgba8(self, pose, rot, W, H, thr, K, row0=0, rows=None, out=None):
        """The viewer's pixels of image rows [row0, row0+rows) -> [rows*W, 4] uint8 (into `out` when given)."""
        rows = H - row0 if rows is None else rows
        p, r = self._pose_rot(pose, rot)
        if out is not None and (out.dtype != torch.uint8 or tuple(out.shape) != (rows * W, 4) or not out.is_contiguous()
                                or out.device != self._dev()):
            raise ValueError("render_camera_rgba8: out must be a contiguous uint8 [rows*W, 4] tensor on the renderer's device")
        out = out if out is not None else torch.empty((rows * W, 4), dtype=torch.uint8, device=self._dev())
        with torch.cuda.device(self.device):
            self._check(self.lib.adn_render_camera_rgba8(self.handle, _fptr(p), _fptr(r), W, H, row0, rows, float(thr), int(K),
                                                         out.data_ptr(), self._stream()))
        return out

    def render_rays_host(self, pose, rot, dirs_np, thr, K, want_nsamples=True, out=None):
        """Host buffers in, host buffers out (H2D / D2H inside the call).  Arrays registered with register_host_buffer
        (or already page-locked) are DMA'd in place; anything else -- including the temporaries a dtype / layout
        conversion creates here -- goes through the context's pinned staging buffers."""
        p, r = self._pose_rot(pose, rot)
        d = np.ascontiguousarray(dirs_np, dtype=np.float32).reshape(-1, 3)
        n = d.shape[0]
        rgb = out if out is not None else np.empty((n, 3), dtype=np.float32)
        ns = np.empty((n,), dtype=np.int32) if want_nsamples else None
        self._check(self.lib.adn_render_rays_host(self.handle, _fptr(p), _fptr(r), d.ctypes.data, n, float(thr), int(K),
                                                  rgb.ctypes.data, ns.ctypes.data if ns is not None else None))
        return dict(rgb=rgb, n_samples=ns)

    def render_camera_host(self, pose, rot, W, H, thr, K, row0=0, rows=None, out=None, want_nsamples=False):
        rows = H - row0 if rows is None else rows
        p, r = self._pose_rot(pose, rot)
        n = rows * W
        rgb = out if out is not None else np.empty((n, 3), dtype=np.float32)
        ns = np.empty((n,), dtype=np.int32) if want_nsamples else None
        self._check(self.lib.adn_render_camera_host(self.handle, _fptr(p), _fptr(r), W, H, row0, rows, float(thr), int(K),
                                                    rgb.ctypes.data, ns.ctypes.data if ns is not None else None))
        return dict(rgb=rgb, n_samples=ns)

    # ---- stage-level entry points (parity tests) --------------------------------------------
    def image_metrics(self, image, reference, clamp01=False):
        """MSE / PSNR of two device images (src/evaluate.py:49-54), reduced on the device."""
        a, b = self._f32(image).reshape(-1), self._f32(reference).reshape(-1)
        if a.numel() != b.numel():
            raise ValueError("image_metrics: shapes differ")
        mse, psnr = C.c_double(), C.c_double()
        with torch.cuda.device(self.device):
            self._check(self.lib.adn_image_metrics(self.handle, a.data_ptr(), b.data_ptr(), a.numel(), int(bool(clamp01)),
                                                   C.byref(mse), C.byref(psnr), self._stream()))
        return dict(mse=mse.value, psnr=psnr.value)

    def flip(self, image, reference, W, H, pixels_per_degree=EVALUATE_PPD, want_map=True):
        """FLIP of two W x H sRGB images (adn_image_flip, src/evaluate.py:119-161): image and reference are [H*W, 3] or
        [H, W, 3] -> dict(mean=float, map=[H, W] float32 on the device, or None when want_map is False).  Waits for the
        current stream first: the call runs on the context's own stream and returns once its results are written.  Refused
        while the current stream captures a CUDA graph (that wait would end the capture)."""
        if torch.cuda.is_current_stream_capturing():
            raise AdnError(1, "flip: the current stream is capturing a CUDA graph; the call synchronises and cannot be captured")
        W, H = int(W), int(H)
        if W < 1 or H < 1:
            raise ValueError("flip: W and H must be >= 1")
        for name, t in (("image", image), ("reference", reference)):
            if tuple(t.shape) not in ((H * W, 3), (H, W, 3)):
                raise ValueError(f"flip: {name} must be [H*W, 3] or [H, W, 3] with W={W}, H={H}, got {tuple(t.shape)}")
        if tuple(image.shape) != tuple(reference.shape):
            raise ValueError("flip: image and reference shapes differ")
        a, b = self._f32(image), self._f32(reference)
        fmap = torch.empty((H, W), dtype=torch.float32, device=self._dev()) if want_map else None
        mean = C.c_double()
        with torch.cuda.device(self.device):
            torch.cuda.current_stream().synchronize()
            self._check(self.lib.adn_image_flip(self.handle, a.data_ptr(), b.data_ptr(), W, H, float(pixels_per_degree),
                                                fmap.data_ptr() if fmap is not None else None, C.byref(mean)))
        return dict(mean=mean.value, map=fmap)

    def iw_ssim(self, image, reference, W, H, layout="evaluate"):
        """IW-SSIM of image (distorted) against reference (original) (adn_image_iwssim, src/evaluate.py:81-88) ->
        dict(score=float, scales=[wmcs of scales 1..5]).  layout "evaluate": [H*W, 3] or [H, W, 3] fp32 as evaluate.py holds
        its images, converted by its rgb2gray(x.view(W, H, -1)); layout "gray": [H*W] or [H, W] planes on the metric's 0-255
        scale.  W, H >= 161.  Waits for the current stream first: the call runs on the context's own stream and returns
        once its results are on the host.  Refused while the current stream captures a CUDA graph."""
        W, H = int(W), int(H)
        if layout not in IWSSIM_LAYOUTS:
            raise ValueError(f"iw_ssim: layout must be one of {sorted(IWSSIM_LAYOUTS)}, got {layout!r}")
        if W < IWSSIM_MIN_SIZE or H < IWSSIM_MIN_SIZE:
            raise ValueError(f"iw_ssim: W and H must be >= {IWSSIM_MIN_SIZE}, got W={W}, H={H}")
        shapes = ((H * W, 3), (H, W, 3)) if layout == "evaluate" else ((H * W,), (H, W))
        for name, t in (("image", image), ("reference", reference)):
            if tuple(t.shape) not in shapes:
                raise ValueError(f"iw_ssim: {name} must be {' or '.join(map(str, shapes))} for layout {layout!r} with "
                                 f"W={W}, H={H}, got {tuple(t.shape)}")
        if tuple(image.shape) != tuple(reference.shape):
            raise ValueError("iw_ssim: image and reference shapes differ")
        if torch.cuda.is_current_stream_capturing():
            raise AdnError(1, "iw_ssim: the current stream is capturing a CUDA graph; the call synchronises and cannot be "
                              "captured")
        a, b = self._f32(image), self._f32(reference)
        score, scales = C.c_double(), (C.c_double * 5)()
        with torch.cuda.device(self.device):
            torch.cuda.current_stream().synchronize()
            self._check(self.lib.adn_image_iwssim(self.handle, a.data_ptr(), b.data_ptr(), W, H, IWSSIM_LAYOUTS[layout],
                                                  C.byref(score), scales))
        return dict(score=score.value, scales=list(scales))

    def generate_ray_directions(self, W, H, row0=0, rows=None):
        rows = H - row0 if rows is None else rows
        out = torch.empty((rows * W, 3), dtype=torch.float32, device=self._dev())
        self._check(self.lib.adn_generate_ray_directions(self.handle, W, H, row0, rows, out.data_ptr(), self._stream()))
        return out

    def stage0(self, pose, rot, dirs):
        p, r = self._pose_rot(pose, rot)
        d = self._f32(dirs).reshape(-1, 3)
        n = d.shape[0]
        x0 = torch.empty((n, self.n_feat0), dtype=torch.float32, device=self._dev())
        ro = torch.empty((n, 3), dtype=torch.float32, device=self._dev())
        rd = torch.empty((n, 3), dtype=torch.float32, device=self._dev())
        self._check(self.lib.adn_stage0_features(self.handle, _fptr(p), _fptr(r), d.data_ptr(), n, x0.data_ptr(),
                                                 ro.data_ptr(), rd.data_ptr(), self._stream()))
        return x0, ro, rd

    def mlp0(self, x0, n_out=None):
        x = self._f32(x0)
        width = self.net_dims(0)[1]              # the library writes [N, n_out of the network that is set]
        if n_out is not None and int(n_out) != width:
            raise ValueError(f"mlp0: the sampling net has {width} outputs, not {n_out}")
        out = torch.empty((x.shape[0], width), dtype=torch.float32, device=self._dev())
        self._check(self.lib.adn_mlp0_forward(self.handle, x.data_ptr(), x.shape[0], out.data_ptr(), self._stream()))
        return out

    def stage2(self, raw0, thr, K):
        """Stage 2 alone (adn_stage2_sample): raw0 [N,D] (D = depth_cells()) -> the packed selection."""
        x = self._f32(raw0)
        if x.dim() != 2 or x.shape[1] != self.depth_cells():
            raise ValueError(f"stage2: raw0 must be [N, {self.depth_cells()}] (the sampling net's depth cells), got {tuple(x.shape)}")
        n = x.shape[0]
        dev = self._dev()
        count = torch.empty((n,), dtype=torch.int32, device=dev)
        offset = torch.empty((n,), dtype=torch.int32, device=dev)
        cap = max(n * K, 1)
        cell = torch.full((cap,), -1, dtype=torch.int32, device=dev)
        ray = torch.full((cap,), -1, dtype=torch.int32, device=dev)
        z = torch.full((cap,), float("nan"), dtype=torch.float32, device=dev)
        zp = torch.full((cap,), float("nan"), dtype=torch.float32, device=dev)
        total = torch.zeros((1,), dtype=torch.int64, device=dev)
        self._check(self.lib.adn_stage2_sample(self.handle, x.data_ptr(), n, float(thr), int(K), count.data_ptr(), offset.data_ptr(),
                                               cell.data_ptr(), ray.data_ptr(), z.data_ptr(), zp.data_ptr(), total.data_ptr(),
                                               self._stream()))
        m = int(total.item())
        return dict(count=count, offset=offset, cell=cell[:m], ray=ray[:m], z=z[:m], zp=zp[:m], total=m)

    def pdf_sample(self, raw0, K, transform=1):
        """FromClassifiedDepth's sample placement alone (adn_pdf_sample): raw0 [N,128] -> dict(count [N], offset [N],
        ray [N K] int32, z [N K] float32 world depth).  transform: 1 = sigmoid, 2 = softmax (option "pdf_transform").
        Waits for the current stream first: the call runs on the context's own stream and returns once its outputs are
        written."""
        x = self._f32(raw0)
        n, dev = x.shape[0], self._dev()
        count = torch.full((n,), -1, dtype=torch.int32, device=dev)
        offset = torch.full((n,), -1, dtype=torch.int32, device=dev)
        ray = torch.full((max(n * K, 1),), -1, dtype=torch.int32, device=dev)
        z = torch.full((max(n * K, 1),), float("nan"), dtype=torch.float32, device=dev)
        with torch.cuda.device(self.device):
            torch.cuda.current_stream().synchronize()
            self._check(self.lib.adn_pdf_sample(self.handle, x.data_ptr(), n, int(K), int(transform), count.data_ptr(),
                                                offset.data_ptr(), ray.data_ptr(), z.data_ptr()))
        return dict(count=count, offset=offset, ray=ray[:n * K], z=z[:n * K])

    def stage5_density(self, raw1, z, ray_d, K, aux=True, rgba8=False):
        """nerf_raw2outputs alone (adn_stage5_density_composite): raw1 [N K, 4], z [N K] and ray_d [N,3] ->
        dict(rgb [N,3], rgba8 [N,4] uint8 when asked, and the aux outputs: True or an iterable of AUX_KEYS).  Synchronises
        like pdf_sample."""
        dev = self._dev()
        r1, zz, rd = self._f32(raw1), self._f32(z), self._f32(ray_d)
        n = rd.shape[0]
        keys = self.AUX_KEYS if aux is True else tuple(aux or ())
        out = dict(rgb=torch.empty((n, 3), dtype=torch.float32, device=dev),
                   rgba8=torch.empty((n, 4), dtype=torch.uint8, device=dev) if rgba8 else None)
        a = AuxOutputs()
        for k in keys:
            if k not in self.AUX_KEYS:
                raise KeyError(f"unknown stage-5 output {k!r}")
            out[k] = torch.empty((n, int(K)) if k in ("weights", "alpha", "z_vals") else (n,), dtype=torch.float32, device=dev)
            setattr(a, "d_" + k, out[k].data_ptr())
        with torch.cuda.device(self.device):
            torch.cuda.current_stream().synchronize()
            self._check(self.lib.adn_stage5_density_composite(self.handle, r1.data_ptr(), zz.data_ptr(), rd.data_ptr(), n, int(K),
                                                              out["rgb"].data_ptr(), out["rgba8"].data_ptr() if rgba8 else None,
                                                              C.byref(a)))
        return out

    def camera_rays(self, pose, rot, dirs, want_ray_dirs=True):
        """The rays of option "sampler" = 2 (adn_camera_rays): dirs [N,3] -> dict(ray_o [N,3] = pose, ray_d [N,3] = R d,
        which stage3 reads, and ray_dirs [N,3], the directions whose norm stage5_density scales its distances by: ray_d, or
        on NDC scenes ndc_rays' un-normalised direction).  Waits for the current stream first, like pdf_sample."""
        p, r = self._pose_rot(pose, rot)
        d = self._f32(dirs).reshape(-1, 3)
        n, dev = d.shape[0], self._dev()
        out = {k: torch.empty((n, 3), dtype=torch.float32, device=dev) for k in ("ray_o", "ray_d")}
        out["ray_dirs"] = torch.empty((n, 3), dtype=torch.float32, device=dev) if want_ray_dirs else None
        with torch.cuda.device(self.device):
            torch.cuda.current_stream().synchronize()
            self._check(self.lib.adn_camera_rays(self.handle, _fptr(p), _fptr(r), d.data_ptr(), n, out["ray_o"].data_ptr(),
                                                 out["ray_d"].data_ptr(), out["ray_dirs"].data_ptr() if want_ray_dirs else None))
        return out

    def linear_depths(self, K):
        """The K depths option "sampler" = 2 places on every ray (adn_linear_depths) -> [K] float32 on the device.  Waits for
        the current stream first, like pdf_sample."""
        z = torch.empty((int(K),), dtype=torch.float32, device=self._dev())
        with torch.cuda.device(self.device):
            torch.cuda.current_stream().synchronize()
            self._check(self.lib.adn_linear_depths(self.handle, int(K), z.data_ptr()))
        return z

    def budget_threshold(self, raw0, thr_min, K, max_samples, out=None):
        """raw0 [N,D] (D = depth_cells()) -> [1] float32 device tensor: the smallest threshold >= thr_min at which stage 2 with K samples per
        ray yields at most max_samples samples (the selection a "sample_budget" render makes).  Stream ordered, no sync."""
        x = self._f32(raw0)
        if x.dim() != 2 or x.shape[1] != self.depth_cells():
            raise ValueError(f"budget_threshold: raw0 must be [N, {self.depth_cells()}] (the sampling net's depth cells), got {tuple(x.shape)}")
        t = out if out is not None else torch.empty((1,), dtype=torch.float32, device=self._dev())
        self._check(self.lib.adn_budget_threshold(self.handle, x.data_ptr(), x.shape[0], float(thr_min), int(K), int(max_samples),
                                                  t.data_ptr(), self._stream()))
        return t

    def sampling_view(self, raw0, rgb=True, rgba8=True):
        """The sampling network's view of raw0 [N,128] (adn_sampling_view, the viewer's render-oracle picture) ->
        dict(rgb [N,3] float32, rgba8 [N,4] uint8); an output asked for with False is None.  Waits for the current stream
        first: the call runs on the context's own stream and returns once its outputs are written.  Refused while the
        current stream captures a CUDA graph (that wait would end the capture)."""
        if torch.cuda.is_current_stream_capturing():
            raise AdnError(1, "sampling_view: the current stream is capturing a CUDA graph; the call synchronises and cannot "
                              "be captured")
        x = self._f32(raw0)
        if x.dim() != 2 or x.shape[1] != 128:
            raise ValueError("sampling_view: raw0 must be [N, 128]")
        n, dev = x.shape[0], self._dev()
        out = dict(rgb=torch.empty((n, 3), dtype=torch.float32, device=dev) if rgb else None,
                   rgba8=torch.empty((n, 4), dtype=torch.uint8, device=dev) if rgba8 else None)
        ptr = lambda t: t.data_ptr() if t is not None else None
        with torch.cuda.device(self.device):
            torch.cuda.current_stream().synchronize()
            self._check(self.lib.adn_sampling_view(self.handle, x.data_ptr(), n, ptr(out["rgb"]), ptr(out["rgba8"])))
        return out

    def stage3(self, ray_o, ray_d, ray_idx, z):
        ro, rd, zz = self._f32(ray_o), self._f32(ray_d), self._f32(z)
        ri = ray_idx.to(device=self._dev(), dtype=torch.int32).contiguous()
        m = zz.shape[0]
        x1 = torch.empty((m, self.n_feat1), dtype=torch.float32, device=self._dev())
        self._check(self.lib.adn_stage3_encode(self.handle, ro.data_ptr(), rd.data_ptr(), ri.data_ptr(), zz.data_ptr(), m,
                                               x1.data_ptr(), self._stream()))
        return x1

    def mlp1(self, x1):
        x = self._f32(x1)
        out = torch.empty((x.shape[0], 4), dtype=torch.float32, device=self._dev())
        self._check(self.lib.adn_mlp1_forward(self.handle, x.data_ptr(), x.shape[0], out.data_ptr(), self._stream()))
        return out

    def stage5(self, raw1, zp, z, offset, count, K, want_aux=True, aux=None, dense=False, rgba8=False, out=None):
        """Stage 5 alone (adn_stage5_composite_aux) -> dict(rgb [N,3], rgba8 [N,4] uint8, and each requested aux output).
        want_aux: weights and depth_map (aux=None only).  aux: True or an iterable of AUX_KEYS.  dense: zp is raw0 [N,K]
        and z / offset / count may be None (K must be 128 or depth_cells()).  out: dict of tensors to write into instead of new ones (keys
        "rgb", "rgba8" and AUX_KEYS; each one given is also requested) -- slots the kernel does not write keep their
        contents."""
        dev = self._dev()
        out = dict(out or {})
        r1, zpp = self._f32(raw1), self._f32(zp)
        n = zpp.shape[0] if dense else count.shape[0]
        zz = self._f32(z) if z is not None else None
        off = offset.to(device=dev, dtype=torch.int32).contiguous() if offset is not None else None
        cnt = count.to(device=dev, dtype=torch.int32).contiguous() if count is not None else None
        keys = (("weights", "depth_map") if want_aux else ()) if aux is None else self.AUX_KEYS if aux is True else tuple(aux)
        keys = tuple(k for k in self.AUX_KEYS if k in keys or k in out)
        shapes = dict(rgb=((n, 3), torch.float32), rgba8=((n, 4), torch.uint8))
        shapes.update({k: ((n, int(K)) if k in ("weights", "alpha", "z_vals") else (n,), torch.float32) for k in self.AUX_KEYS})
        for k in ("rgb",) + (("rgba8",) if rgba8 or "rgba8" in out else ()) + keys:
            if k not in shapes:
                raise KeyError(f"unknown stage-5 output {k!r}")
            shape, dt = shapes[k]
            if k in out:
                t = out[k]
                if t.dtype != dt or tuple(t.shape) != shape or not t.is_contiguous() or t.device != dev:
                    raise ValueError(f"stage5: out[{k!r}] must be a contiguous {dt} {list(shape)} tensor on the renderer's device")
            else:
                out[k] = torch.empty(shape, dtype=dt, device=dev)
        a = AuxOutputs()
        for k in keys:
            setattr(a, "d_" + k, out[k].data_ptr())
        ptr = lambda t: t.data_ptr() if t is not None else None
        with torch.cuda.device(self.device):
            self._check(self.lib.adn_stage5_composite_aux(self.handle, r1.data_ptr(), zpp.data_ptr(), ptr(zz), ptr(off), ptr(cnt),
                                                          n, int(K), int(bool(dense)), out["rgb"].data_ptr(),
                                                          ptr(out.get("rgba8")), C.byref(a), self._stream()))
        if aux is None:
            for k in ("weights", "depth_map"):
                out.setdefault(k, None)
        return out


def _device_tensor(ptr, shape, typestr, device):
    """A torch tensor aliasing device memory owned by the library (__cuda_array_interface__)."""
    class _Holder:
        pass
    h = _Holder()
    h.__cuda_array_interface__ = dict(shape=tuple(shape), typestr=typestr, data=(int(ptr), False), version=3, strides=None)
    return torch.as_tensor(h, device=device)


_RENDERERS = {}


def _fingerprint(net):
    """Changes whenever a parameter tensor is replaced or modified in place (torch bumps `_version` on in-place writes)."""
    sd = net.state_dict() if hasattr(net, "state_dict") else net
    return tuple((k, v.data_ptr(), v._version, tuple(v.shape)) if isinstance(v, torch.Tensor) else (k, id(v)) for k, v in sd.items())


def render(rays, sampling_net, shading_net, adaptiveSamplingThreshold, *, K, scene, device=0):
    """The public entry named by BASELINE.json.  `rays` = dict(pose [3], rot [3,3], dirs [N,3]) -- the
    three tensors `TrainConfig.inference` reads from its batch (ImagePose, ImageRotation,
    RayDirectionsSamples; src/features.py:832-834).  Returns (rgb [N,3], n_samples [N]).

    Like the reference's inference() it always renders with the CURRENT parameters: the packed device copy of the two
    networks is cached, but the cache entry holds the networks themselves (their ids cannot be recycled) and is
    re-packed whenever a parameter tensor was replaced or written in place since the last call."""
    key = (device, tuple(sorted((k, str(v)) for k, v in scene.items())))
    entry = _RENDERERS.get(key)
    fp = (_fingerprint(sampling_net), _fingerprint(shading_net))
    if entry is None or entry["nets"][0] is not sampling_net or entry["nets"][1] is not shading_net:
        if entry is not None:
            entry["renderer"].close()
        _RENDERERS.clear()
        entry = dict(renderer=Renderer(scene, device=device, sampling_net=sampling_net, shading_net=shading_net),
                     nets=(sampling_net, shading_net), fp=fp)
        _RENDERERS[key] = entry
    elif entry["fp"] != fp:
        if entry["fp"][0] != fp[0]:
            entry["renderer"].set_weights(0, sampling_net)
        if entry["fp"][1] != fp[1]:
            entry["renderer"].set_weights(1, shading_net)
        entry["fp"] = fp
    out = entry["renderer"].render_rays(rays["pose"], rays["rot"], rays["dirs"], adaptiveSamplingThreshold, K)
    return out["rgb"], out["n_samples"]
