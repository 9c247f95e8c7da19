"""Loading of the explicit-ray fixtures (tests/golden/make_golden_rays.py): the seeded scene, weights and the stored rays."""
import torch

from keypointnerf_b200 import synthetic as syn
from tests.util import checksum, load_golden

RAY_CASES = ["rays_ortho", "rays_mixed"]


def load_rays_case(name):
    """(golden arrays, meta, scene, weights, origins, dirs, near_far) of a ray fixture; the rays as torch CPU tensors."""
    g, meta, sha = load_golden(name)
    scene = syn.make_scene(src_size=meta["src_size"], n_views=meta["n_views"], n_kpt=meta["n_kpt"], seed=meta["scene_seed"],
                           fg_mode=meta["fg_mode"], fg_hole=meta["fg_hole"])
    weights = syn.make_weights(meta["n_kpt"], seed=meta["w_seed"])
    assert checksum(scene, weights) == sha, "seeded inputs drifted from the ones the golden run used"
    return g, meta, scene, weights, torch.from_numpy(g["rays_o"]), torch.from_numpy(g["rays_d"]), torch.from_numpy(g["near_far"])
