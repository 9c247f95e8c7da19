"""Drop-in ``KeypointNeRF`` for the reference's volumetric-rendering hot path.

Mirrors the Python surface the reference's Lightning module calls (SURVEY.md section 8b):
``KeypointNeRF(cfg)`` with the same sub-module names / ``state_dict`` keys for the
hot-path networks (reference ``src/model.py:559-609``), ``query`` (690), and the static
``render_pifu_nerf`` (897) / ``batch_render_pifu_nerf`` (942) entry points with the same
positional order and ``**config`` keys.  All per-sample arithmetic runs in the CUDA
library behind ``include/kpnerf_b200.h``; this file only marshals tensors.

The 2-D image encoders (``geo_encoder``, ``tex_encoder``; ``keypointnerf_b200/encoders.py``) carry the
reference's parameter names, run channels-last and hand their outputs to the kernels without a
re-layout pass; their feature maps are cached per source-image set.  A reference checkpoint loads
with ``strict=True`` (``vgg_loss.*`` entries, which only the training loss reads, are accepted and
dropped).  Out of scope (SURVEY.md section 8f.3): the training ``forward``.
"""
from __future__ import annotations

import copy
import math

import torch
import torch.nn as nn

from . import encoders as enc
from .renderer import RayMarcher
from .synthetic import layer_table


class _WNLinear(nn.Module):
    """Parameter holder with the keys of ``weight_norm(nn.Linear)`` (reference ``src/utils.py:542-543``):
    ``linear.bias``, ``linear.weight_g`` (out,1), ``linear.weight_v`` (out,in)."""

    class _P(nn.Module):
        def __init__(self, n_in, n_out, wn):
            super().__init__()
            self.bias = nn.Parameter(torch.zeros(n_out))
            if wn:
                v = torch.empty(n_out, n_in)
                nn.init.kaiming_uniform_(v, a=5 ** 0.5)
                self.weight_g = nn.Parameter(v.norm(dim=1, keepdim=True))
                self.weight_v = nn.Parameter(v)
            else:
                w = torch.empty(n_out, n_in)
                nn.init.kaiming_normal_(w, a=0, mode="fan_in", nonlinearity="relu")
                self.weight = nn.Parameter(w)

    def __init__(self, n_in, n_out, wn):
        super().__init__()
        self.linear = self._P(n_in, n_out, wn)


class _LayerStack(nn.Module):
    def __init__(self, dims_in, dims_out):
        super().__init__()
        n = len(dims_out)
        self.layers = nn.ModuleList([_WNLinear(i, o, wn=(k != n - 1)) for k, (i, o) in enumerate(zip(dims_in, dims_out))])


class MLPUNetFusion(nn.Module):
    """Parameters of the geometry MLP (reference ``src/utils.py:476-517``): ``layers1`` (per-view
    MLP-UNet with feature skips) and ``layers2`` (density head after view pooling)."""

    def __init__(self, n_dims1, n_dims2, skip_dims, skip_layers, nl_layer="softplus", norm="weight",
                 pool_types=("mean", "var"), **kwargs):
        super().__init__()
        if nl_layer != "softplus" or norm != "weight" or list(pool_types) != ["mean", "var"]:
            raise NotImplementedError("only the configs/zju.json geometry MLP (softplus, weight norm, mean+var) is built")
        skip = {j: skip_dims[i] for i, j in enumerate(skip_layers)}
        d_in = [n_dims1[i] + skip.get(i, 0) for i in range(len(n_dims1) - 1)]
        self.pool = nn.Module()
        self.layers1 = _LayerStack(d_in, n_dims1[1:])
        self.layers2 = _LayerStack(n_dims2[:-1], n_dims2[1:])


class IBRRenderingHead(nn.Module):
    """Parameters of the colour-blending head (reference ``src/model.py:1239-1258``)."""

    def __init__(self, in_channels=32, **kwargs):
        super().__init__()
        c = in_channels + 3
        self.ani_al = nn.Parameter(torch.tensor(0.2))
        seq = lambda *dims: nn.Sequential(*[m for i in range(len(dims) - 1)
                                            for m in (nn.Linear(dims[i], dims[i + 1]), nn.ELU(inplace=True))])
        self.ray_encoder = seq(4, 16, c)
        self.base_layer = seq(c * 3, 64, 32)
        self.vis_layer1 = seq(32, 32, 33)
        self.vis_layer2 = nn.Sequential(nn.Linear(32, 32), nn.ELU(inplace=True), nn.Linear(32, 1), nn.Sigmoid())
        self.out_layer = nn.Sequential(nn.Linear(37, 16), nn.ELU(inplace=True), nn.Linear(16, 8), nn.ELU(inplace=True),
                                       nn.Linear(8, 1))


class SpatialEncoder(nn.Module):
    """Hyper-parameters of the relative keypoint encoding (reference ``src/spatial.py:9-21``)."""

    def __init__(self, sp_level, sp_type, scale, n_kpt, **kwargs):
        super().__init__()
        if sp_type != "rel_z_decay":
            raise NotImplementedError(f"sp_type={sp_type!r}: only 'rel_z_decay' (configs/zju.json:41) is built")
        self.sp_type, self.sp_level, self.n_kpt, self.scale = sp_type, sp_level, n_kpt, scale
        self.kwargs = kwargs
        self.register_buffer("center", torch.tensor(kwargs.get("center", [0.0, 0.0, 0.0])).float())

    def get_dim(self):
        return (1 + 2 * self.sp_level) * self.n_kpt


_HOT_MODULES = ("mlp_geo", "mlp_tex", "ibr_compress_gfeat")


class KeypointNeRF(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        model_cfg = cfg["models"]["KeypointNeRF"]
        self.train_out_h = model_cfg.get("train_out_h", 64)
        self.train_out_w = model_cfg.get("train_out_w", 64)
        self.disable_fg_mask = model_cfg.get("disable_fg_mask", False)
        self.sp_encoder = SpatialEncoder(**model_cfg["sp_args"])
        geo_args = copy.deepcopy(model_cfg["mlp_geo_args"])
        geo_args["n_dims1"][0] = self.sp_encoder.get_dim()
        self.mlp_geo = MLPUNetFusion(**geo_args)
        self.mlp_tex = IBRRenderingHead(**model_cfg["mlp_tex_args"]["args"])
        self.ibr_compress_gfeat = nn.Linear(model_cfg["mlp_tex_args"]["gcompress"]["in_ch"],
                                            model_cfg["mlp_tex_args"]["gcompress"]["out_ch"])
        # image encoders (reference src/model.py:575,598): built when the config describes them, channels-last
        self.geo_encoder = enc.to_channels_last(enc.HGFilterV2(**model_cfg["geo_args"])) if "geo_args" in model_cfg else None
        self.tex_encoder = enc.to_channels_last(enc.ResBlkEncoder(**model_cfg["tex_args"])) if "tex_args" in model_cfg else None
        self._geo_cache, self._tex_cache = enc.FeatureCache(), enc.FeatureCache()
        self.sp_encoder_postfusion = None
        self.ds_geo = model_cfg.get("ds_geo", 0)
        self.ds_tex = model_cfg.get("ds_tex", 0)
        self.v_level = model_cfg.get("v_level", 0)
        self.dr_level = model_cfg.get("dr_level", 5)
        self.feat_geo = None
        self.feat_tex = None
        self.kwargs = model_cfg
        self.vgg_loss = None
        self.disable_bg = True
        self._marcher = None
        self._w_key = None
        self._scene_key = None
        self._last_bounds = None
        self.engine = 0   # kpn_opts.engine: 0 tensor cores (default), 1 fp32 CUDA cores, 2-4 variants (include/kpnerf_b200.h)

    # ---- feature caching (reference src/model.py:642-688) -----------------------------------------
    def attach_im_feat(self, im, return_val=False):
        if return_val:
            out = {"feat_geo": self.attach_geo_feat(im, True)}
            ft = self.attach_tex_feat(im, True)
            if ft is not None:
                out["feat_tex"] = ft
            return out
        self.attach_geo_feat(im)
        self.attach_tex_feat(im)

    @staticmethod
    def _encode(module, im, n_down, grad=False):
        """avg-pool ``n_down`` times, map [0,1] -> [-1,1], run the encoder channels-last (with autograd when ``grad``); the
        outputs' storage is [V][H][W][C], the layout the kernels gather from (no re-layout pass in kpn_set_scene)."""
        if im.dim() == 5:
            im = im.view(-1, *im.shape[2:])
        x = im.contiguous(memory_format=torch.channels_last)
        for _ in range(n_down):
            x = torch.nn.functional.avg_pool2d(x, 2, stride=2)
        with torch.set_grad_enabled(grad):
            out = module(2.0 * x - 1.0)
        return [enc.nhwc_view(o) for o in out] if isinstance(out, (list, tuple)) else enc.nhwc_view(out)

    def attach_geo_feat(self, im, return_val=False):
        """Reference ``src/model.py:653-667``.  The maps of the last source-image set are cached: the reference re-runs the
        encoders for every rendered camera (``src/model.py:913-914`` after 479), a camera sweep here runs them once."""
        if self.geo_encoder is None:
            raise RuntimeError("this model was built without geo_args: pass feat_geo explicitly")
        if not return_val:
            self.im = im.clone()
        feat = self._geo_cache.get(im, lambda x: self._encode(self.geo_encoder, x, self.ds_geo))
        if return_val:
            return feat
        self.feat_geo = feat

    def attach_tex_feat(self, im, return_val=False):
        """Reference ``src/model.py:669-680``."""
        if self.tex_encoder is None:
            return None
        feat = self._tex_cache.get(im, lambda x: self._encode(self.tex_encoder, x, self.ds_tex))
        if return_val:
            return feat
        self.feat_tex = feat

    def detach_im_feat(self):
        self.feat_geo = None
        self.feat_tex = None
        self._geo_cache.clear()
        self._tex_cache.clear()

    def train(self, mode: bool = True):
        self._geo_cache.clear()    # the encoder weights may change between calls while training
        self._tex_cache.clear()
        return super().train(mode)

    # ---- checkpoints (reference load_ckpt: strict load_state_dict, src/model.py:113-117) ----------
    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        # The reference's model also owns vgg_loss (a frozen VGG19 the training loss reads, src/model.py:608) and, in some
        # configs, encoders this instance was built without: accept those entries and drop them, so that a strict load of a
        # reference checkpoint succeeds.  Everything the render path uses is still checked strictly.
        ignored = ["vgg_loss.", "sp_encoder_postfusion."]
        if self.geo_encoder is None:
            ignored.append("geo_encoder.")
        if self.tex_encoder is None:
            ignored.append("tex_encoder.")
        for k in [k for k in state_dict if k.startswith(prefix) and k[len(prefix):].startswith(tuple(ignored))]:
            del state_dict[k]
        self._geo_cache.clear()
        self._tex_cache.clear()
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)

    # ---- marshalling -----------------------------------------------------------------------------
    def _device_index(self):
        p = self.ibr_compress_gfeat.weight
        if not p.is_cuda:
            raise RuntimeError("KeypointNeRF must live on a CUDA device (.cuda()): the ray-march path has no CPU fallback")
        return p.device.index if p.device.index is not None else torch.cuda.current_device()

    def marcher(self) -> RayMarcher:
        dev = self._device_index()
        if self._marcher is None or self._marcher.device != dev:
            self._marcher = RayMarcher(dev)
            self._w_key = None
            self._scene_key = None
        hot = {}
        for name in _HOT_MODULES:   # only the networks the ray-march reads (not the 28 M encoder parameters)
            for k, v in getattr(self, name).state_dict().items():
                hot[f"{name}.{k}"] = v
        key = tuple((k, v.data_ptr(), v._version) for k, v in hot.items())
        if key != self._w_key:
            sp = self.sp_encoder
            self._marcher.set_weights(hot, n_kpt=sp.n_kpt, sp_level=sp.sp_level, sp_scale=sp.scale,
                                      sp_sigma=sp.kwargs.get("sigma", 150.0))
            self._w_key = key
            self._scene_key = None
        return self._marcher

    def marcher_dtype(self) -> str:
        """Arithmetic type of the dense layers in the selected engine."""
        sp = self.sp_encoder
        tc = self.engine != 1
        return "fp16 operands, fp32 accumulate (wgmma)" if tc else "fp32"

    def _bind_scene(self, cam, feat_geo, feat_tex, sp_data, img, fg_mask, bounds):
        m = self.marcher()
        tensors = [cam["KRT"], sp_data["extrin"], sp_data["kpt3d"], bounds, feat_geo[0], feat_geo[1], feat_tex, img]
        if fg_mask is not None:
            tensors.append(fg_mask)
        key = tuple((t.data_ptr(), t._version, tuple(t.shape)) for t in tensors) + (
            float(cam["width"]), float(cam["height"]), float(cam["znear"]), float(cam["zfar"]))
        if key != self._scene_key:
            m.set_scene(KRT=cam["KRT"], extrin=sp_data["extrin"], kpt3d=sp_data["kpt3d"].reshape(-1, 3), bounds=bounds,
                        feat64=feat_geo[0], feat8=feat_geo[1], feat_tex=feat_tex, img=img,
                        fg=None if self.disable_fg_mask else fg_mask,
                        width=cam["width"], height=cam["height"], znear=cam["znear"], zfar=cam["zfar"],
                        nml_scale=cam.get("nml_scale", 100.0))
            self._scene_key = key
        self._last_bounds = bounds
        return m

    def invalidate_scene(self):
        """Force the next render/query to re-bind the scene (the cache key is tensor identity + version: call this after
        writing into a bound tensor through a view that does not bump its version)."""
        self._scene_key = None

    # ---- query (reference src/model.py:690-782) --------------------------------------------------
    def query(self, pts, cam, feat_geo=None, feat_tex=None, n_views=1, sp_data={}, tx_data={}, view=None,
              n_pts_samples=-1, **kwargs):
        """Returns ``(out (B,N,5) = [sdf_raw, rad, r, g, b], valid (B,N,1) bool)``; B must be 1."""
        assert pts.shape[0] == 1, "batch size 1 only (the reference's bbox test already requires it, src/model.py:1191)"
        feat_geo = self.feat_geo if feat_geo is None else feat_geo
        feat_tex = self.feat_tex if feat_tex is None else feat_tex
        bounds = kwargs.get("bounds")
        if bounds is None:   # query does not read the bounds; reuse whatever the bound scene has so that it is not re-packed
            bounds = self._last_bounds if self._last_bounds is not None else torch.zeros(1, 2, 3)
        m = self._bind_scene(cam, feat_geo, feat_tex, sp_data, tx_data["img"], kwargs.get("src_foreground_mask"), bounds)
        out, valid = m.query(pts[0], view[0], engine=self.engine)
        return out[None], valid[None, :, None]

    def forward(self, *args, **kwargs):
        raise NotImplementedError("the training forward (autograd through the ray-march) is outside this build's "
                                  "scope (SURVEY.md section 8f.3); use the reference implementation to train")

    # ---- full frame (reference src/model.py:897-940) ---------------------------------------------
    @staticmethod
    def render_pifu_nerf(net, img_in, cam_in, cam_tar, level=5, sp_data={}, bkg_emb=None, camcenter=None,
                         objcenter=None, tar_img=None, **config):
        """Same contract as the reference: dict of detached CPU tensors ``(C,H,W)``.  The reference
        renders stride^2 strided 64x64-style passes and pixel-shuffles them; rays are independent, so
        this renders the frame in ONE launch sequence with no per-pass host synchronisation."""
        config = dict(config)
        feat_geo = config.pop("feat_geo", None)
        feat_tex = config.pop("feat_tex", None)
        shard = config.pop("dist_shard", None)   # extension: (rank, world) -> this rank renders one lattice phase of the frame
        if feat_geo is None:
            feat_geo = net.attach_geo_feat(img_in, return_val=True)
        if feat_tex is None:
            feat_tex = net.attach_tex_feat(img_in, return_val=True)
        if shard is not None and shard[1] > 1:
            out = KeypointNeRF._render_sharded(net, img_in, cam_in, cam_tar, tar_img, feat_geo, feat_tex, sp_data, shard, **config)
        else:
            out = KeypointNeRF._render(net, img_in, cam_in, cam_tar, 1, 0, 0, tar_img, feat_geo, feat_tex, sp_data,
                                       out_device="cpu", **config)
        ret = {}
        for k, v in out.items():
            if v is None or v.dim() < 3:
                continue
            ret[k] = v[0] if v.dim() == 4 else v  # (B,C,h,w) -> (C,h,w); (B,h,w) -> (1,h,w) like the reference
        if "tex_fg_fine" not in ret:
            # fine=False: the reference's caller reads tex_fg_fine unconditionally (_arrange_nerf_images, src/model.py:428)
            ret["tex_fg_fine"] = ret["tex_fg"]
        return ret

    @staticmethod
    def _render_sharded(net, img_in, cam_in, cam_tar, tar_img, feat_geo, feat_tex, sp_data, shard, **config):
        """One frame over ``world`` ranks (BASELINE config 4): lattice phase per rank, ONE all-gather per plane, host copy."""
        from . import distributed as D
        rank, world = shard
        width = int(cam_tar.get("width", cam_in["width"]))
        height = int(cam_tar.get("height", cam_in["height"]))
        fine = config.get("fine", False)
        m = net._bind_scene(cam_in, feat_geo, feat_tex, sp_data, img_in, config.get("src_foreground_mask"), config["bounds"])
        res = D.render_frame_lattice_sharded(m, K=cam_tar["K"], RT=cam_tar["RT"], znear=cam_tar.get("znear", cam_in["znear"]),
                                             zfar=cam_tar.get("zfar", cam_in["zfar"]), width=width, height=height, rank=rank,
                                             world=world, S_c=config.get("sample_per_ray_c", 64),
                                             S_f=config.get("sample_per_ray_f", 64), fine=fine, engine=net.engine,
                                             ert_eps=config.get("ert_eps", 0.0))
        keys = ["tex_fg", "depth", "alpha"] + (["tex_fg_fine", "depth_fine", "alpha_fine", "sdf"] if fine else [])
        out = {k: res[k].cpu()[None] for k in keys}
        if tar_img is not None:
            out["tar_img"] = tar_img.cpu()
        return out

    # ---- camera sweep (reference KeypointNeRFLightningModule.render_novel_views, src/model.py:475-507) ------------
    @staticmethod
    def render_views(net, img_in, cam_in, cams_tar, sp_data={}, rank=0, world=1, **config):
        """Render one source-image set from many target cameras (the 90-camera sweep of ``render_dynamic.py``;
        SURVEY.md section 8f.2).  Same ``**config`` keys and per-frame result dicts (detached CPU tensors) as
        ``render_pifu_nerf``, but the encoders run once, the scene is bound once, every frame is enqueued without a host
        synchronisation and its device-to-host copy runs on a side stream into pinned memory while the next frame renders;
        the call synchronises once at the end.  ``rank``/``world``: this process renders cameras ``rank::world`` (one process
        per GPU; the caller gathers the frames it wants, e.g. with ``distributed.gather_views``)."""
        config = dict(config)
        feat_geo = config.pop("feat_geo", None)
        feat_tex = config.pop("feat_tex", None)
        if feat_geo is None:
            feat_geo = net.attach_geo_feat(img_in, return_val=True)
        if feat_tex is None:
            feat_tex = net.attach_tex_feat(img_in, return_val=True)
        dev = torch.device("cuda", net._device_index())
        main, side = torch.cuda.current_stream(dev), torch.cuda.Stream(dev)
        frames, inflight = [], []
        for cam_tar in list(cams_tar)[rank::world]:
            out = KeypointNeRF._render(net, img_in, cam_in, cam_tar, 1, 0, 0, None, feat_geo, feat_tex, sp_data,
                                       out_device="cuda", **config)
            done = torch.cuda.Event()
            done.record(main)
            host = {}
            with torch.cuda.stream(side):
                side.wait_event(done)
                for k, v in out.items():
                    h = torch.empty(v.shape[1:] if v.dim() == 4 else v.shape, dtype=v.dtype, pin_memory=True)
                    h.copy_(v[0] if v.dim() == 4 else v, non_blocking=True)
                    host[k] = h
            inflight.append(out)     # the device planes must outlive their copies
            if "tex_fg_fine" not in host:
                host["tex_fg_fine"] = host["tex_fg"]
            frames.append(host)
        side.synchronize()
        net.marcher().check_health()
        return frames

    # ---- surface extraction (the reference's users run query on a grid + skimage.measure.marching_cubes) -------------
    @staticmethod
    def mesh_grid(bounds, resolution=256):
        """The grid ``extract_mesh`` samples: spacing ``h = max extent / (resolution - 1)`` on every axis,
        ``n_a = ceil(extent_a / h - 1e-6) + 1`` points along axis a, origin ``bounds[0]``.  Returns (origin, spacing, dims) as
        Python floats / ints, dims = (nx, ny, nz)."""
        b = torch.as_tensor(bounds).detach().reshape(2, 3).double().cpu()
        lo, ext = b[0], b[1] - b[0]
        if resolution < 2 or not bool(torch.all(ext > 0)):
            raise ValueError("extract_mesh needs resolution >= 2 and bounds[1] > bounds[0] on every axis")
        h = float(ext.max()) / (resolution - 1)
        dims = tuple(int(math.ceil(float(e) / h - 1e-6)) + 1 for e in ext)
        return tuple(float(x) for x in lo), (h, h, h), dims

    @staticmethod
    def extract_mesh(net, img_in, cam_in, sp_data, bounds, level, resolution=256, colors=True, src_foreground_mask=None,
                     feat_geo=None, feat_tex=None):
        """The subject's surface as a triangle mesh: the density ``valid * relu(rad)`` (reference ``src/model.py:978-997``; it
        depends only on the point, being pooled over the source views) on ``mesh_grid(bounds, resolution)`` with ``net.engine``,
        zero-padded by one voxel so that the surface closes at the box, then marching cubes at ``level`` on the device.
        ``colors``: the RGB of ``query`` at every vertex seen along ``-normal``.  Returns a dict of device tensors:
        ``vertices`` (V,3), ``faces`` (F,3) int32 (counter-clockwise seen from outside), ``normals`` (V,3) and ``colors`` (V,3)."""
        if feat_geo is None:
            feat_geo = net.attach_geo_feat(img_in, return_val=True)
        if feat_tex is None:
            feat_tex = net.attach_tex_feat(img_in, return_val=True)
        m = net._bind_scene(cam_in, feat_geo, feat_tex, sp_data, img_in, src_foreground_mask, bounds)
        origin, spacing, dims = KeypointNeRF.mesh_grid(bounds, resolution)
        out, valid = m.query_grid(origin, spacing, dims, engine=net.engine)
        field = torch.nn.functional.pad(out[..., 1].clamp_min(0.0) * valid, (1, 1, 1, 1, 1, 1))
        porigin = tuple(o - h for o, h in zip(origin, spacing))
        verts, faces, normals = m.marching_cubes(field, porigin, spacing, level, normals=True)
        res = {"vertices": verts, "faces": faces, "normals": normals}
        if colors:   # an empty mesh (level above every density) has no vertices to query
            res["colors"] = m.query(verts, -normals, engine=net.engine)[0][:, 2:5] if verts.shape[0] else verts.new_zeros(0, 3)
        return res

    # ---- one pass (reference src/model.py:942-1108) ----------------------------------------------
    @staticmethod
    def batch_render_pifu_nerf(net, img_in, cam_in, n_views, cam_tar, level=2, stride=0, tar_img=None, feat_geo=None,
                               feat_tex=None, sp_data={}, objcenter=None, **config):
        if net.training:
            raise NotImplementedError("training branch (random patch, jitter, view dropout) is outside this build's scope")
        assert img_in.shape[0] // n_views == 1, "batch size 1 only"
        if feat_geo is None:
            feat_geo = net.attach_geo_feat(img_in, return_val=True)
        if feat_tex is None:
            feat_tex = net.attach_tex_feat(img_in, return_val=True)
        step = 2 ** (level - 1)
        if isinstance(stride, int):
            assert stride < step
            x_off = y_off = stride
        elif isinstance(stride, torch.Tensor):
            sv = stride.reshape(-1).tolist()
            assert max(sv) < step
            x_off, y_off = int(sv[0]), int(sv[1])
        else:
            raise NotImplementedError("unsupported stride type")
        return KeypointNeRF._render(net, img_in, cam_in, cam_tar, step, x_off, y_off, tar_img, feat_geo, feat_tex,
                                    sp_data, out_device=None, **config)

    @staticmethod
    def _check_config(config):
        """The eval-branch options this build renders; the training-time ones raise."""
        if not config.get("uniform", False):
            raise NotImplementedError("uniform=False (stratified jitter of the sample depths, the default of dr_kwargs in "
                                      "configs/zju.json) is a training-time option outside this build: pass uniform=True, as the "
                                      "reference's own render/validation/test callers do (src/model.py:463)")
        if config.get("separate_cf", False):
            raise NotImplementedError("separate_cf (separate coarse/fine heads) is outside this build")
        if config.get("rand_noise_std", 0.0) > 0.0:
            raise NotImplementedError("rand_noise_std > 0 (density noise, dr_kwargs.rand_noise_std of configs/zju.json) is a "
                                      "training-time option outside this build: the reference's render callers do not pass it "
                                      "(src/model.py:453-473)")

    @staticmethod
    def _render(net, img_in, cam_in, cam_tar, step, x_off, y_off, tar_img, feat_geo, feat_tex, sp_data, out_device,
                **config):
        S_c = config.get("sample_per_ray_c", 64)
        S_f = config.get("sample_per_ray_f", 64)
        fine = config.get("fine", False)
        KeypointNeRF._check_config(config)
        width = int(cam_tar.get("width", cam_in["width"]))
        height = int(cam_tar.get("height", cam_in["height"]))
        znear = cam_tar.get("znear", cam_in["znear"])
        zfar = cam_tar.get("zfar", cam_in["zfar"])
        assert width % step == 0 and height % step == 0
        nx, ny = width // step, height // step
        m = net._bind_scene(cam_in, feat_geo, feat_tex, sp_data, img_in, config.get("src_foreground_mask"), config["bounds"])
        res = m.render(K=cam_tar["K"], RT=cam_tar["RT"], znear=znear, zfar=zfar, x0=x_off, y0=y_off, step=step,
                       nx=nx, ny=ny, S_c=S_c, S_f=S_f, fine=fine, out_device=out_device, engine=net.engine,
                       ert_eps=config.get("ert_eps", 0.0))
        out = {"tex_fg": res["tex_fg"][None], "depth": res["depth"][None], "alpha": res["alpha"][None]}
        if fine:
            out.update({"tex_fg_fine": res["tex_fg_fine"][None], "depth_fine": res["depth_fine"][None],
                        "alpha_fine": res["alpha_fine"][None], "sdf": res["sdf"][None]})
        if tar_img is not None:  # reference src/model.py:1097-1107
            with torch.no_grad():
                ys = torch.arange(y_off, height, step, device=tar_img.device)
                xs = torch.arange(x_off, width, step, device=tar_img.device)
                sub = tar_img[:, :, ys][:, :, :, xs]
                out["tar_img"] = sub.to(out["tex_fg"].device)
                if "msk" in config:
                    msk = config["msk"].reshape(1, 1, height, width)
                    out["tar_alpha"] = msk[:, :, ys][:, :, :, xs].float().to(out["tex_fg"].device)
        return out

    # ---- explicit rays (the eval branch of src/model.py:1038-1096 on given rays) ------------------------------------------
    @staticmethod
    def render_rays(net, img_in, cam_in, rays_o, rays_d, near_far, sp_data={}, **config):
        """Render explicit rays: ``rays_o``, ``rays_d`` (n,3) (unit directions, used as given) and ``near_far`` (n,2) (before the
        clip to ``config["bounds"]``), e.g. the pixels of a ``mask_at_box``, an orthographic bundle or the rays of several
        cameras at once.  Same ``**config`` keys as ``render_pifu_nerf``.  Returns ``tex_fg`` (3,n), ``depth`` / ``alpha`` (n,)
        (and with ``fine``: ``tex_fg_fine``, ``depth_fine``, ``alpha_fine``, ``sdf``) on the rays' device; ray i equals the
        pixel of ``render_pifu_nerf`` whose ray it is, bit for bit."""
        config = dict(config)
        feat_geo = config.pop("feat_geo", None)
        feat_tex = config.pop("feat_tex", None)
        KeypointNeRF._check_config(config)
        if feat_geo is None:
            feat_geo = net.attach_geo_feat(img_in, return_val=True)
        if feat_tex is None:
            feat_tex = net.attach_tex_feat(img_in, return_val=True)
        fine = config.get("fine", False)
        m = net._bind_scene(cam_in, feat_geo, feat_tex, sp_data, img_in, config.get("src_foreground_mask"), config["bounds"])
        res = m.render_rays(rays_o, rays_d, near_far, S_c=config.get("sample_per_ray_c", 64), S_f=config.get("sample_per_ray_f", 64),
                            fine=fine, engine=net.engine, ert_eps=config.get("ert_eps", 0.0),
                            out_device="cuda" if rays_o.is_cuda else "cpu")
        keys = ["tex_fg", "depth", "alpha"] + (["tex_fg_fine", "depth_fine", "alpha_fine", "sdf"] if fine else [])
        return {k: res[k] for k in keys}

    # ---- differentiable explicit rays ---------------------------------------------------------------------------------------
    def hot_parameters(self):
        """The parameters the ray-march reads, in the order of ``synthetic.layer_table``: per layer (weight_v, weight_g, bias) of a
        weight-normed layer or (weight, bias) of a plain one, then ``mlp_tex.ani_al``."""
        named = dict(self.named_parameters())
        out = []
        for name, _, _, wn in layer_table(self.sp_encoder.n_kpt, self.sp_encoder.sp_level):
            out += [named[name + s] for s in ((".weight_v", ".weight_g", ".bias") if wn else (".weight", ".bias"))]
        return out + [self.mlp_tex.ani_al]

    @staticmethod
    def render_rays_grad(net, img_in, cam_in, rays_o, rays_d, near_far, sp_data={}, **config):
        """``render_rays`` with outputs that carry a ``grad_fn``: ``loss.backward()`` reaches every hot-path parameter
        (``hot_parameters``) and the feature maps ``feat_geo[0]``, ``feat_geo[1]``, ``feat_tex`` (the gradients are computed by
        ``kpn_render_rays_backward``: fp32 CUDA cores, the reference's autograd semantics of the eval branch).  Same keys,
        refusals and outputs as ``render_rays``; the forward runs on ``net.engine``.  Without ``feat_geo`` / ``feat_tex`` the
        encoders run here with autograd (and without the feature cache), so that the gradient reaches them too.  The fine
        pass' depths, the source images, cameras, keypoints, bounds, rays and masks get no gradient."""
        config = dict(config)
        feat_geo = config.pop("feat_geo", None)
        feat_tex = config.pop("feat_tex", None)
        KeypointNeRF._check_config(config)
        if config.get("ert_eps", 0.0) > 0.0:
            raise NotImplementedError("ert_eps > 0: the samples early-ray termination skips have gradients")
        if feat_geo is None:
            if net.geo_encoder is None:
                raise RuntimeError("this model was built without geo_args: pass feat_geo explicitly")
            feat_geo = KeypointNeRF._encode(net.geo_encoder, img_in, net.ds_geo, grad=True)
        if feat_tex is None:
            if net.tex_encoder is None:
                raise RuntimeError("this model was built without tex_args: pass feat_tex explicitly")
            feat_tex = KeypointNeRF._encode(net.tex_encoder, img_in, net.ds_tex, grad=True)
        fine = config.get("fine", False)
        keys = ["tex_fg", "depth", "alpha"] + (["tex_fg_fine", "depth_fine", "alpha_fine", "sdf"] if fine else [])
        opts = dict(S_c=config.get("sample_per_ray_c", 64), S_f=config.get("sample_per_ray_f", 64), fine=fine)
        fg = config.get("src_foreground_mask")
        bind = lambda: net._bind_scene(cam_in, feat_geo, feat_tex, sp_data, img_in, fg, config["bounds"])
        outs = _RenderRays.apply(net, bind, (rays_o, rays_d, near_far), opts, keys, feat_geo[0], feat_geo[1], feat_tex,
                                 *net.hot_parameters())
        return dict(zip(keys, outs))


def param_grads(net, g, params):
    """The gradients of ``hot_parameters`` (``params``, in that order) from ``RayMarcher.render_rays_backward``'s ``g``: the folded
    weight ``W = g v / ||v||`` of a weight-normed layer maps per row to ``dg = sum_k dW v / ||v||``,
    ``dv = (g / ||v||) (dW - (dW . v^) v^)``."""
    out, i = [], 0
    for l, (_, _, _, wn) in enumerate(layer_table(net.sp_encoder.n_kpt, net.sp_encoder.sp_level)):
        dW, db = g["dW"][l], g["db"][l]
        if wn:
            v, gw = params[i], params[i + 1]
            nrm = v.norm(dim=1, keepdim=True)
            vh = v / nrm
            proj = (dW * vh).sum(1, keepdim=True)
            out += [(gw / nrm) * (dW - proj * vh), proj.to(gw.dtype), db]
            i += 3
        else:
            out += [dW, db]
            i += 2
    out.append(g["d_ani_al"].reshape(params[i].shape))
    return out


class _RenderRays(torch.autograd.Function):
    """Forward: ``RayMarcher.render_rays`` on ``net.engine``; backward: ``RayMarcher.render_rays_backward`` at the fine depths the
    forward resampled (its outputs' own), then ``param_grads``.  First order only."""

    @staticmethod
    def forward(ctx, net, bind, rays, opts, keys, feat64, feat8, feat_tex, *params):
        m = bind()
        res = m.render_rays(*rays, **opts, engine=net.engine, debug=opts["fine"],
                            out_device="cuda" if rays[0].is_cuda else "cpu")
        ctx.net, ctx.bind, ctx.rays, ctx.opts, ctx.keys = net, bind, rays, opts, keys
        ctx.z_fine = res.get("z_fine")
        ctx.save_for_backward(*params)
        return tuple(res[k] for k in keys)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, *grads):
        m = ctx.bind()
        g = m.render_rays_backward(*ctx.rays, {k: v for k, v in zip(ctx.keys, grads) if v is not None}, **ctx.opts,
                                   z_fine_override=ctx.z_fine)
        maps = [g["d_feat64"], g["d_feat8"], g["d_feat_tex"]]
        return (None, None, None, None, None, *maps, *param_grads(ctx.net, g, ctx.saved_tensors))
