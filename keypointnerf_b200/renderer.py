"""RayMarcher: the host-side handle on one device's ray-march context (C ABI, ctypes).

It accepts torch tensors (CUDA tensors are passed as device pointers on the current
stream; CPU tensors as host pointers, the library then does the H2D/D2H copies itself)
and mirrors the argument meaning of the reference's ``KeypointNeRF.query`` /
``batch_render_pifu_nerf`` (reference ``src/model.py:690-782, 942-1108``).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _lib as L
from .synthetic import layer_table


# Host outputs: pinned (fast asynchronous D2H, but a cold pinned allocation costs milliseconds) or pageable.  KPN_PINNED_OUT=0/1.
_PINNED_OUT = os.environ.get("KPN_PINNED_OUT", "1") != "0"


def _f32c(t: torch.Tensor) -> torch.Tensor:
    t = t.detach()
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


class RayMarcher:
    def __init__(self, device: int | torch.device | None = None):
        self.lib = L.load()
        if device is None:
            device = torch.cuda.current_device()
        if isinstance(device, torch.device):
            device = device.index if device.index is not None else torch.cuda.current_device()
        self.device = int(device)
        self.ctx = C.c_void_p()
        rc = self.lib.kpn_create(self.device, C.byref(self.ctx))
        if rc != L.KPN_OK:
            raise L.KpnError(f"kpn_create(device={self.device}) failed with status {rc} "
                             "(a CUDA device is required; there is no CPU fallback)")
        self._keep = []       # tensors that must outlive the asynchronous calls of the current scene
        self.n_views = 0
        self.n_kpt, self.sp_level = 0, 3                                  # of the weights set last
        self.map_shapes = [(0, 64, 1, 1), (0, 8, 1, 1), (0, 8, 1, 1)]      # (V, C, H, W) of the bound scene's gathered maps

    def close(self):
        if getattr(self, "ctx", None) is not None and self.ctx.value:
            self.lib.kpn_destroy(self.ctx)
            self.ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self) -> C.c_void_p:
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # ---- weights -------------------------------------------------------------------------------
    def set_weights(self, state: dict, n_kpt: int, sp_level: int = 3, sp_scale: float = 1.0, sp_sigma: float = 0.1):
        """``state`` maps the reference's parameter names (no ``model.`` prefix) to tensors/arrays."""
        w = L.KpnWeights()
        keep = []

        def host(x):
            a = x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
            a = np.ascontiguousarray(a, dtype=np.float32)
            keep.append(a)
            return a

        for i, (name, n_out, n_in, wn) in enumerate(layer_table(n_kpt)):
            lay = w.layer[i]
            if wn:
                v, g = host(state[name + ".weight_v"]), host(state[name + ".weight_g"])
                lay.w, lay.g = v.ctypes.data, g.ctypes.data
                shape = v.shape
            else:
                m = host(state[name + ".weight"])
                lay.w, lay.g = m.ctypes.data, None
                shape = m.shape
            b = host(state[name + ".bias"])
            lay.bias = b.ctypes.data
            lay.n_out, lay.n_in = int(shape[0]), int(shape[1])
        w.ani_al = float(np.asarray(host(state["mlp_tex.ani_al"])).reshape(-1)[0])
        w.n_kpt, w.sp_level, w.sp_scale, w.sp_sigma = int(n_kpt), int(sp_level), float(sp_scale), float(sp_sigma)
        L.check(self.lib, self.ctx, self.lib.kpn_set_weights(self.ctx, C.byref(w)), "kpn_set_weights")
        self.n_kpt, self.sp_level = int(n_kpt), int(sp_level)

    # ---- scene ---------------------------------------------------------------------------------
    def set_scene(self, *, KRT, extrin, kpt3d, bounds, feat64, feat8, feat_tex, img, fg, width, height,
                  znear=2.0, zfar=5.0, nml_scale=100.0):
        on_dev = bool(img.is_cuda)
        dev = img.device

        def prep(t):
            t = _f32c(t)
            return t if t.device == dev else t.to(dev)

        layout = 0

        def prep_map(t, bit):
            # feature maps that are already stored [V][H][W][C] (channels-last encoder outputs) are taken as they are
            nonlocal layout
            t = t.detach()
            if t.dtype == torch.float32 and t.device == dev and t.dim() == 4 and t.shape[1] > 1 \
                    and t.is_contiguous(memory_format=torch.channels_last):
                layout |= bit
                return t
            return prep(t)

        KRT, extrin = prep(KRT).reshape(-1, 4, 4), prep(extrin).reshape(-1, 4, 4)
        kpt3d, bounds = prep(kpt3d).reshape(-1, 3), prep(bounds).reshape(2, 3)
        feat64, feat8 = prep_map(feat64, L.KPN_NHWC_FEAT64), prep_map(feat8, L.KPN_NHWC_FEAT8)
        feat_tex, img = prep_map(feat_tex, L.KPN_NHWC_FEATTEX), prep(img)
        V = img.shape[0]
        s = L.KpnScene()
        s.n_views, s.n_kpt = V, kpt3d.shape[0]
        s.src_width, s.src_height = float(width), float(height)
        s.znear, s.zfar, s.nml_scale = float(znear), float(zfar), float(nml_scale)
        s.KRT, s.extrin, s.kpt3d, s.bounds = KRT.data_ptr(), extrin.data_ptr(), kpt3d.data_ptr(), bounds.data_ptr()
        s.feat64, (s.f64_c, s.f64_h, s.f64_w) = feat64.data_ptr(), feat64.shape[1:]
        s.feat8, (s.f8_c, s.f8_h, s.f8_w) = feat8.data_ptr(), feat8.shape[1:]
        s.feat_tex, (s.ftex_c, s.ftex_h, s.ftex_w) = feat_tex.data_ptr(), feat_tex.shape[1:]
        s.img, (s.img_h, s.img_w) = img.data_ptr(), img.shape[2:]
        keep = [KRT, extrin, kpt3d, bounds, feat64, feat8, feat_tex, img]
        if fg is not None:
            fg8 = fg.detach().reshape(V, 1, *fg.shape[-2:]).to(device=dev, dtype=torch.uint8).contiguous()
            s.fg, s.fg_h, s.fg_w = fg8.data_ptr(), fg8.shape[2], fg8.shape[3]
            keep.append(fg8)
        else:
            s.fg = None
        s.mem = L.KPN_MEM_DEVICE if on_dev else L.KPN_MEM_HOST
        s.layout = layout
        L.check(self.lib, self.ctx, self.lib.kpn_set_scene(self.ctx, C.byref(s), self._stream()), "kpn_set_scene")
        self._keep = keep
        self.n_views = V
        self.map_shapes = [tuple(feat64.shape), tuple(feat8.shape), tuple(feat_tex.shape)]

    # ---- render --------------------------------------------------------------------------------
    def reserve(self, max_rays: int, max_samples: int):
        """Pre-size the workspace so that later renders of at most this size never allocate (``kpn_reserve``)."""
        L.check(self.lib, self.ctx, self.lib.kpn_reserve(self.ctx, int(max_rays), int(max_samples)), "kpn_reserve")

    def check_health(self):
        """Raise if a tensor-core kernel's barrier wait gave up since the last check (``kpn_check_health``)."""
        L.check(self.lib, self.ctx, self.lib.kpn_check_health(self.ctx, self._stream()), "kpn_check_health")

    @staticmethod
    def _target(K, RT, znear, zfar, x0, y0, step, nx, ny, step_y):
        K, RT = _f32c(K).reshape(-1, 4, 4)[0].contiguous(), _f32c(RT).reshape(-1, 4, 4)[0].contiguous()
        if RT.device != K.device:
            RT = RT.to(K.device)
        tg = L.KpnTarget()
        tg.K, tg.RT = K.data_ptr(), RT.data_ptr()
        tg.znear, tg.zfar = float(znear), float(zfar)
        tg.x0, tg.y0, tg.step, tg.nx, tg.ny, tg.step_y = int(x0), int(y0), int(step), int(nx), int(ny), int(step_y)
        tg.mem = L.KPN_MEM_DEVICE if K.is_cuda else L.KPN_MEM_HOST
        return tg, [K, RT]

    def _march(self, call, what, shape, out_device, S_c, S_f, fine, engine, z_fine_override, debug, ert_eps, keep) -> dict:
        """One kpn_render / kpn_render_rays call ``call(opts, out)`` whose rays form an image of ``shape`` ((ny, nx) or (n,))."""
        op = L.KpnOpts()
        op.sample_per_ray_c, op.sample_per_ray_f, op.fine = int(S_c), int(S_f), int(bool(fine))
        op.ert_eps, op.engine = float(ert_eps), int(engine)
        host_out = str(out_device).startswith("cpu")
        odev = torch.device("cpu") if host_out else torch.device("cuda", self.device)
        n = int(np.prod(shape))

        def alloc(*shape):
            if host_out:   # fresh host tensors per call, like the reference's .cpu() (src/model.py:929)
                return torch.empty(*shape, dtype=torch.float32, pin_memory=_PINNED_OUT)
            return torch.empty(*shape, dtype=torch.float32, device=odev)

        res = {"tex_fg": alloc(3, *shape), "depth": alloc(*shape), "alpha": alloc(*shape)}
        if fine:
            res.update({"tex_fg_fine": alloc(3, *shape), "depth_fine": alloc(*shape), "alpha_fine": alloc(*shape),
                        "sdf": alloc(*shape)})
            if debug:
                res["z_fine"] = alloc(n, S_c + S_f)
        if debug:
            res["contrib"] = alloc(n, S_c)
        if z_fine_override is not None:
            zo = _f32c(z_fine_override).to(odev).contiguous()
            assert zo.numel() == n * (S_c + S_f)
            op.z_fine_override = zo.data_ptr()
            keep.append(zo)
        out = L.KpnOut()
        for k, v in res.items():
            setattr(out, k, v.data_ptr())
        out.mem = L.KPN_MEM_HOST if host_out else L.KPN_MEM_DEVICE
        L.check(self.lib, self.ctx, call(C.byref(op), C.byref(out)), what)
        self._keep_call = keep
        if host_out:  # results are host tensors: make them readable on return (reference does .cpu(), src/model.py:929)
            torch.cuda.current_stream(self.device).synchronize()
            self.check_health()   # the watchdog words travelled with the results: a tripped barrier wait raises here
        return res

    def render(self, *, K, RT, znear, zfar, x0, y0, step, nx, ny, S_c, S_f=0, fine=False, out_device=None,
               engine=0, z_fine_override=None, debug=False, ert_eps=0.0, step_y=0) -> dict:
        """One ``kpn_render`` call.  Returns planar tensors on ``out_device`` ('cuda' or 'cpu';
        default: where K lives)."""
        tg, keep = self._target(K, RT, znear, zfar, x0, y0, step, nx, ny, step_y)
        if out_device is None:
            out_device = "cuda" if keep[0].is_cuda else "cpu"
        call = lambda op, out: self.lib.kpn_render(self.ctx, C.byref(tg), op, out, self._stream())
        return self._march(call, "kpn_render", (ny, nx), out_device, S_c, S_f, fine, engine, z_fine_override, debug, ert_eps, keep)

    def camera_rays(self, *, K, RT, znear, zfar, x0=0, y0=0, step=1, nx, ny, step_y=0):
        """The rays ``render`` marches for the same lattice (``kpn_camera_rays``): ``(origins (n,3), dirs (n,3), near_far (n,2))``
        on K's device, ray ``j*nx + i`` for pixel (i, j), near/far before the bounding-box clip.  Needs no weights or scene."""
        tg, keep = self._target(K, RT, znear, zfar, x0, y0, step, nx, ny, step_y)
        n = int(nx) * int(ny)
        on_dev = keep[0].is_cuda
        kw = dict(device=keep[0].device) if on_dev else dict(pin_memory=True)
        o = torch.empty(n, 3, dtype=torch.float32, **kw)
        d = torch.empty(n, 3, dtype=torch.float32, **kw)
        nf = torch.empty(n, 2, dtype=torch.float32, **kw)
        L.check(self.lib, self.ctx,
                self.lib.kpn_camera_rays(self.ctx, C.byref(tg), o.data_ptr(), d.data_ptr(), nf.data_ptr(),
                                         L.KPN_MEM_DEVICE if on_dev else L.KPN_MEM_HOST, self._stream()), "kpn_camera_rays")
        self._keep_call = keep
        if not on_dev:
            torch.cuda.current_stream(self.device).synchronize()
        return o, d, nf

    def render_rays(self, origins, dirs, near_far, *, S_c, S_f=0, fine=False, engine=0, ert_eps=0.0, out_device=None,
                    z_fine_override=None, debug=False) -> dict:
        """One ``kpn_render_rays`` call on explicit rays: ``origins``, ``dirs`` (n,3) (unit directions, used as given),
        ``near_far`` (n,2) before the bounding-box clip.  Returns the dict of ``render`` with every (ny, nx) plane shaped (n,),
        on ``out_device`` (default: where ``origins`` lives)."""
        o = _f32c(origins).reshape(-1, 3)
        d, nf = _f32c(dirs).reshape(-1, 3), _f32c(near_far).reshape(-1, 2)
        d, nf = d.to(o.device).contiguous(), nf.to(o.device).contiguous()
        n = o.shape[0]
        if d.shape[0] != n or nf.shape[0] != n:
            raise ValueError(f"render_rays: {n} origins, {d.shape[0]} directions, {nf.shape[0]} near/far pairs")
        if out_device is None:
            out_device = "cuda" if o.is_cuda else "cpu"
        rays = L.KpnRays()
        rays.origins, rays.dirs, rays.near_far, rays.n = o.data_ptr(), d.data_ptr(), nf.data_ptr(), n
        rays.mem = L.KPN_MEM_DEVICE if o.is_cuda else L.KPN_MEM_HOST
        call = lambda op, out: self.lib.kpn_render_rays(self.ctx, C.byref(rays), op, out, self._stream())
        return self._march(call, "kpn_render_rays", (n,), out_device, S_c, S_f, fine, engine, z_fine_override, debug, ert_eps,
                           [o, d, nf])

    _GRAD_KEYS = ("tex_fg", "depth", "alpha", "tex_fg_fine", "depth_fine", "alpha_fine", "sdf")

    def render_rays_backward(self, origins, dirs, near_far, grad_out: dict, *, S_c, S_f=0, fine=False, ert_eps=0.0,
                             z_fine_override=None) -> dict:
        """The backward of ``render_rays`` (``kpn_render_rays_backward``): ``grad_out`` maps output names of ``render_rays``
        (``tex_fg`` (3,n), ``depth``, ``alpha`` (n,), with ``fine`` also ``tex_fg_fine``, ``depth_fine``, ``alpha_fine``,
        ``sdf``) to dL/d that output; a missing key is zero.  Returns device tensors on this context's device: ``dW`` and ``db``
        (lists over the layers of ``synthetic.layer_table``, ``dW[l]`` (n_out, n_in) of the folded weight ``g v / ||v||``),
        ``d_ani_al`` (scalar) and ``d_feat64``, ``d_feat8``, ``d_feat_tex`` shaped (V, C, H, W) like the bound maps, stored
        channels-last.  The forward is recomputed with the fp32 engine; the fine depths are constants."""
        dev = torch.device("cuda", self.device)
        o = _f32c(origins).reshape(-1, 3).to(dev).contiguous()
        d, nf = _f32c(dirs).reshape(-1, 3).to(dev).contiguous(), _f32c(near_far).reshape(-1, 2).to(dev).contiguous()
        n = o.shape[0]
        if d.shape[0] != n or nf.shape[0] != n:
            raise ValueError(f"render_rays_backward: {n} origins, {d.shape[0]} directions, {nf.shape[0]} near/far pairs")
        rays = L.KpnRays()
        rays.origins, rays.dirs, rays.near_far, rays.n, rays.mem = o.data_ptr(), d.data_ptr(), nf.data_ptr(), n, L.KPN_MEM_DEVICE
        op = L.KpnOpts()
        op.sample_per_ray_c, op.sample_per_ray_f, op.fine = int(S_c), int(S_f), int(bool(fine))
        op.ert_eps, op.engine = float(ert_eps), 1
        keep = [o, d, nf]
        if z_fine_override is not None:
            zo = _f32c(z_fine_override).to(dev).contiguous()
            assert zo.numel() == n * (S_c + S_f)
            op.z_fine_override = zo.data_ptr()
            keep.append(zo)
        gout = L.KpnOut()
        for k, v in grad_out.items():
            if k not in self._GRAD_KEYS:
                raise ValueError(f"render_rays_backward: no output {k!r}")
            if v is None:
                continue
            g = _f32c(v).to(dev).contiguous()
            if g.numel() != (3 * n if k.startswith("tex_fg") else n):
                raise ValueError(f"render_rays_backward: dL/d{k} has {g.numel()} values for {n} rays")
            setattr(gout, k, g.data_ptr())
            keep.append(g)
        gout.mem = L.KPN_MEM_DEVICE
        gr = L.KpnGrads()
        dW, db = [], []
        for i, (_, n_out, n_in, _) in enumerate(layer_table(self.n_kpt, self.sp_level)):
            dW.append(torch.empty(n_out, n_in, dtype=torch.float32, device=dev))
            db.append(torch.empty(n_out, dtype=torch.float32, device=dev))
            gr.dW[i], gr.db[i] = dW[-1].data_ptr(), db[-1].data_ptr()
        d_ani = torch.empty((), dtype=torch.float32, device=dev)
        maps = [torch.empty(s, dtype=torch.float32, device=dev, memory_format=torch.channels_last) for s in self.map_shapes]
        gr.d_ani_al, gr.d_feat64, gr.d_feat8, gr.d_feat_tex = d_ani.data_ptr(), *(m.data_ptr() for m in maps)
        gr.mem = L.KPN_MEM_DEVICE
        L.check(self.lib, self.ctx, self.lib.kpn_render_rays_backward(self.ctx, C.byref(rays), C.byref(op), C.byref(gout), C.byref(gr),
                                                                       self._stream()), "kpn_render_rays_backward")
        self._keep_call = keep
        return {"dW": dW, "db": db, "d_ani_al": d_ani, "d_feat64": maps[0], "d_feat8": maps[1], "d_feat_tex": maps[2]}

    def query(self, pts: torch.Tensor, view: torch.Tensor, engine: int = 0):
        """``KeypointNeRF.query`` for explicit points: returns out (n,5)=[sdf_raw, rad, r, g, b], valid (n,) bool."""
        pts, view = _f32c(pts).reshape(-1, 3), _f32c(view).reshape(-1, 3)
        n = pts.shape[0]
        on_dev = pts.is_cuda
        if on_dev:
            out = torch.empty(n, 5, dtype=torch.float32, device=pts.device)
            valid = torch.empty(n, dtype=torch.uint8, device=pts.device)
        else:
            out = torch.empty(n, 5, dtype=torch.float32, pin_memory=True)
            valid = torch.empty(n, dtype=torch.uint8, pin_memory=True)
        op = L.KpnOpts()
        op.engine = int(engine)
        L.check(self.lib, self.ctx,
                self.lib.kpn_query(self.ctx, pts.data_ptr(), view.data_ptr(), n, out.data_ptr(), valid.data_ptr(),
                                   L.KPN_MEM_DEVICE if on_dev else L.KPN_MEM_HOST, C.byref(op), self._stream()),
                "kpn_query")
        self._keep_call = [pts, view]
        if not on_dev:
            torch.cuda.current_stream(self.device).synchronize()
            self.check_health()
        return out, valid.bool()

    def query_grid(self, origin, spacing, dims, engine: int = 0):
        """Geometry-only ``query`` on the grid points ``origin + spacing * (i, j, k)`` (``kpn_query_grid``), ``dims`` = (nx, ny, nz).
        Returns ``(out (nz,ny,nx,2) = [sdf_raw, rad], valid (nz,ny,nx) bool)`` on this context's device; the values equal columns
        0-1 of ``query`` at the same points bit for bit."""
        nx, ny, nz = (int(d) for d in dims)
        if min(nx, ny, nz) < 1 or nx * ny * nz > 2 ** 31 - 1:   # refused before the outputs are allocated
            raise L.KpnError(f"query_grid: grid {nx} x {ny} x {nz}: every extent >= 1, at most 2^31 - 1 points")
        g = L.KpnGrid()
        g.origin[:] = [float(x) for x in origin]
        g.spacing[:] = [float(x) for x in spacing]
        g.nx, g.ny, g.nz = nx, ny, nz
        dev = torch.device("cuda", self.device)
        n = nx * ny * nz
        out = torch.empty(n * 2, dtype=torch.float32, device=dev)
        valid = torch.empty(n, dtype=torch.uint8, device=dev)
        op = L.KpnOpts()
        op.engine = int(engine)
        L.check(self.lib, self.ctx,
                self.lib.kpn_query_grid(self.ctx, C.byref(g), out.data_ptr(), valid.data_ptr(), L.KPN_MEM_DEVICE, C.byref(op),
                                        self._stream()), "kpn_query_grid")
        return out.view(nz, ny, nx, 2), valid.view(nz, ny, nx).bool()

    def marching_cubes(self, field: torch.Tensor, origin, spacing, level: float, normals: bool = True):
        """Marching cubes of ``field`` (nz,ny,nx) at ``level`` (inside: f > level) on the grid ``origin + spacing * (i, j, k)``
        (``kpn_mesh_begin`` + ``kpn_mesh_emit``).  Returns ``(vertices (V,3) float32, faces (F,3) int32, normals (V,3) float32
        or None)`` on the field's device (a host field is meshed on this context's device and the results are copied back);
        faces are counter-clockwise seen from the side where f <= level.  Synchronises the current stream once (the counts size
        the outputs)."""
        f = _f32c(field)
        if f.dim() != 3:
            raise ValueError(f"field must be (nz, ny, nx), got {tuple(f.shape)}")
        dev = torch.device("cuda", self.device)
        if f.device != dev:
            f = f.to(dev)
        nz, ny, nx = f.shape
        counts = (C.c_longlong * 2)()
        L.check(self.lib, self.ctx,
                self.lib.kpn_mesh_begin(self.ctx, f.data_ptr(), nx, ny, nz, float(level), counts, self._stream()), "kpn_mesh_begin")
        nv, nf = int(counts[0]), int(counts[1])
        verts = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        nrm = torch.empty(nv, 3, dtype=torch.float32, device=dev) if normals else None
        faces = torch.empty(nf, 3, dtype=torch.int32, device=dev)
        o = (C.c_float * 3)(*[float(x) for x in origin])
        h = (C.c_float * 3)(*[float(x) for x in spacing])
        L.check(self.lib, self.ctx,
                self.lib.kpn_mesh_emit(self.ctx, f.data_ptr(), o, h, verts.data_ptr(), nrm.data_ptr() if normals else None,
                                       faces.data_ptr(), L.KPN_MEM_DEVICE, self._stream()), "kpn_mesh_emit")
        self._keep_call = [f]
        out_dev = field.device
        return verts.to(out_dev), faces.to(out_dev), (nrm.to(out_dev) if normals else None)

    # ---- source-view decode (reference ZJUDataset.__getitem__, src/zju_dataset.py:266-287) ----------
    def decode_views(self, images: torch.Tensor, masks: torch.Tensor | None, K, D, ratio: float = 0.5):
        """Undistort + resize + mask every source view on the device (bit-identical to the reference's cv2 calls).
        ``images`` (V,H0,W0,3) uint8 RGB as read from disk, ``masks`` (V,H0,W0) uint8/bool (non-zero = foreground) or None,
        ``K`` (V,3,3) and ``D`` (V,5) float32 camera matrices / distortion coefficients, ``ratio`` = 1/integer.
        Returns ``(img (V,3,H,W) float32 in [0,1] with the background zeroed, mask (V,1,H,W) bool, K scaled by ratio)`` on the
        device the images live on (host tensors are staged by the library on the current stream)."""
        factor = int(round(1.0 / float(ratio)))
        assert factor >= 1 and abs(factor * float(ratio) - 1.0) < 1e-6, "ratio must be 1 / integer"
        images = images.detach().to(torch.uint8).contiguous()
        V, H0, W0, _ = images.shape
        on_dev = images.is_cuda
        dev = images.device
        if masks is not None:
            masks = masks.detach().to(device=dev, dtype=torch.uint8).reshape(V, H0, W0).contiguous()
        Kn = np.asarray(K.detach().cpu() if isinstance(K, torch.Tensor) else K, dtype=np.float32).reshape(V, 3, 3)
        Dn = np.asarray(D.detach().cpu() if isinstance(D, torch.Tensor) else D, dtype=np.float32).reshape(V, -1)
        cams = np.zeros((V, 18), dtype=np.float64)
        for v in range(V):   # cv2.undistort: newCameraMatrix = K, maps computed in double from the float32 inputs
            Kd = Kn[v].astype(np.float64)
            cams[v, :9] = np.linalg.inv(Kd).reshape(-1)
            cams[v, 9:13] = (Kd[0, 0], Kd[1, 1], Kd[0, 2], Kd[1, 2])
            cams[v, 13:13 + min(5, Dn.shape[1])] = Dn[v, :5].astype(np.float64)
        cams_t = torch.from_numpy(cams)
        cams_t = cams_t.to(dev) if on_dev else cams_t
        H, W = H0 // factor, W0 // factor
        kw = dict(device=dev) if on_dev else dict(pin_memory=True)
        img = torch.empty(V, 3, H, W, dtype=torch.float32, **kw)
        msk = torch.empty(V, 1, H, W, dtype=torch.uint8, **kw)
        L.check(self.lib, self.ctx,
                self.lib.kpn_decode_views(self.ctx, images.data_ptr(), masks.data_ptr() if masks is not None else None,
                                          cams_t.data_ptr(), V, H0, W0, factor, img.data_ptr(), msk.data_ptr(),
                                          L.KPN_MEM_DEVICE if on_dev else L.KPN_MEM_HOST, self._stream()), "kpn_decode_views")
        self._keep_call = [images, masks, cams_t]
        if not on_dev:
            torch.cuda.current_stream(self.device).synchronize()
        K_out = torch.from_numpy(Kn.copy())
        K_out[:, :2] = K_out[:, :2] * float(ratio)          # in_K[:2] = in_K[:2] * self.ratio  (src/zju_dataset.py:296)
        return img, msk.bool(), K_out

    def stats(self) -> dict:
        st = L.KpnStats()
        L.check(self.lib, self.ctx, self.lib.kpn_get_stats(self.ctx, C.byref(st), self._stream()), "kpn_get_stats")
        return {"samples_total": int(st.samples_total), "samples_valid": int(st.samples_valid),
                "kernel_launches": int(st.kernel_launches), "shade_launches": int(st.shade_launches),
                "shade_ms": float(st.shade_ms), "samples_coloured": int(st.samples_coloured), "geo_ms": float(st.geo_ms)}

    def set_profiling(self, enable: bool):
        L.check(self.lib, self.ctx, self.lib.kpn_set_profiling(self.ctx, int(bool(enable))), "kpn_set_profiling")
