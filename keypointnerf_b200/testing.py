"""Helpers shared by tests, smoke and bench: build a model from a weight dict and turn a synthetic
scene (numpy) into the torch argument dicts of the reference API (``decode_batch``,
reference ``src/model.py:309-414``)."""
from __future__ import annotations

import numpy as np
import torch

from . import synthetic as syn
from .config import default_cfg
from .model import KeypointNeRF


def build_model(weights: dict, n_kpt: int, device="cuda:0", sp_args: dict | None = None) -> KeypointNeRF:
    """``sp_args``: overrides of the config's ``sp_level`` / ``scale`` / ``sigma`` (``synthetic.sp_args``; sigma None leaves the
    key out, so the model takes the reference's default of 150)."""
    cfg = default_cfg(n_kpt)
    if sp_args:
        cfg["models"]["KeypointNeRF"]["sp_args"] = syn.sp_args(n_kpt, **sp_args)
    net = KeypointNeRF(cfg)
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in weights.items()}
    res = net.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys, res.unexpected_keys
    missing = [k for k in res.missing_keys if not k.startswith(("sp_encoder", "geo_encoder", "tex_encoder"))]
    assert not missing, missing
    return net.to(device).eval()


def scene_tensors(scene: dict, target: dict, device="cuda:0", pin: bool = False) -> dict:
    def t(a):
        x = torch.from_numpy(np.ascontiguousarray(a))
        if str(device).startswith("cuda"):
            return x.to(device)
        return x.pin_memory() if pin else x

    cam = {"KRT": t(scene["KRT"]), "K": t(scene["K"]), "Rt": t(scene["extrin"]), "extrin": t(scene["extrin"]),
           "znear": scene["znear"], "zfar": scene["zfar"], "width": scene["width"], "height": scene["height"],
           "nml_scale": scene["nml_scale"]}
    cam_tar = {"K": t(target["K"]), "RT": t(target["RT"]), "KRT": t(target["KRT"]), "width": target["width"],
               "height": target["height"], "znear": target["znear"], "zfar": target["zfar"],
               "nml_scale": target["nml_scale"]}
    return {
        "cam": cam, "cam_tar": cam_tar,
        "sp_data": {"extrin": t(scene["extrin"]), "kpt3d": t(scene["kpt3d"])},
        "feat_geo": [t(scene["feat64"]), t(scene["feat8"])],
        "feat_tex": t(scene["feat_tex"]), "img": t(scene["img"]), "fg": t(scene["fg"]), "bounds": t(scene["bounds"]),
    }
