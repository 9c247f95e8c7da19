"""CPU-side checks: the C-ABI library loads and exports every symbol include/kpnerf_b200.h declares,
the ctypes struct mirrors match the header's field order, and the host module keeps the reference's
state_dict keys.  No compute calls (no GPU here)."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import __graft_entry__ as G
from keypointnerf_b200 import _lib as L
from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200.config import default_cfg
from keypointnerf_b200.model import KeypointNeRF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "kpnerf_b200.h")).read()


@pytest.fixture(scope="module")
def lib():
    G.build()
    return L.load()


def test_every_declared_symbol_is_exported(lib):
    declared = set(re.findall(r"^(?:int|void|const char\*)\s+(kpn_\w+)\(", HEADER, flags=re.M))
    assert declared == set(L.EXPORTS)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.kpn_abi_version() == int(re.search(r"#define KPN_ABI_VERSION (\d+)", HEADER).group(1))


def _header_fields(struct_name):
    body = re.search(r"typedef struct \{((?:(?!typedef struct).)*?)\} " + struct_name + r";", HEADER, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for stmt in body.split(";"):
        stmt = stmt.strip()
        if not stmt:
            continue
        for p in stmt.split(","):
            names.append(re.findall(r"(\w+)(?:\[\w+\])?\s*$", p.strip())[0])
    return names


@pytest.mark.parametrize("cname,ctype", [("kpn_layer", L.KpnLayer), ("kpn_weights", L.KpnWeights),
                                         ("kpn_scene", L.KpnScene), ("kpn_target", L.KpnTarget),
                                         ("kpn_opts", L.KpnOpts), ("kpn_out", L.KpnOut), ("kpn_stats", L.KpnStats)])
def test_ctypes_mirrors_header(cname, ctype):
    assert _header_fields(cname) == [f[0] for f in ctype._fields_]


def test_create_fails_loudly_without_gpu(lib):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    ctx = C.c_void_p()
    assert lib.kpn_create(0, C.byref(ctx)) != 0 and not ctx.value
    from keypointnerf_b200.renderer import RayMarcher
    with pytest.raises(RuntimeError):
        RayMarcher(0)


def test_state_dict_keys_match_reference_names():
    for n_kpt in (18, 24):
        net = KeypointNeRF(default_cfg(n_kpt))
        sd = net.state_dict()
        w = syn.make_weights(n_kpt)
        hot = {k: v for k, v in sd.items() if k.startswith(("mlp_geo", "mlp_tex", "ibr_compress"))}
        assert set(hot) == set(w), set(hot) ^ set(w)
        for k, v in w.items():
            assert tuple(hot[k].shape) == tuple(np.asarray(v).shape), k
        assert "sp_encoder.center" in sd
        net.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in w.items()}, strict=False)


def test_no_cpu_fallback_in_model():
    net = KeypointNeRF(default_cfg(18))
    with pytest.raises(RuntimeError):
        net.marcher()  # parameters on CPU -> must refuse, not fall back
    with pytest.raises(NotImplementedError):
        net.forward()


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "keypointnerf_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, flags=re.M), f


@pytest.mark.parametrize("n_kpt", [18, 24])
def test_tensor_core_input_permutation_is_a_bijection(lib, n_kpt):
    """Geometry-stage weight packing (host code of the library, no GPU): every input of a stage is multiplied with its own K
    index, the bias row has a K index of its own, everything fits the padded K; layer 0 additionally keeps the two column runs
    (thread 0 | thread 1) aligned as the activation-tile stores of the kernel require."""
    n_in = {0: 7 * n_kpt + 64, 1: 128, 2: 136, 3: 120, 4: 128, 5: 64}
    for stage, n in n_in.items():
        kmap = (C.c_int * n)()
        kbias, kpad = C.c_int(), C.c_int()
        assert lib.kpn_debug_kmap(stage, n_kpt, n, kmap, C.byref(kbias), C.byref(kpad)) == 0
        ks = list(kmap)
        assert len(set(ks)) == n and kbias.value not in ks
        assert 0 <= min(ks) and max(ks + [kbias.value]) < kpad.value and kpad.value % 16 == 0
    # layer 0: encoding element (r, k) of keypoint pair j = k // 2 sits at packed column 7 j' + r, pairs of one thread contiguous
    kmap = (C.c_int * (7 * n_kpt + 64))()
    lib.kpn_debug_kmap(0, n_kpt, 7 * n_kpt + 64, kmap, None, None)
    cols = np.array(kmap) // 2
    for k in range(0, n_kpt, 2):
        pair_cols = sorted(cols[r * n_kpt + k] for r in range(7))
        assert pair_cols == list(range(pair_cols[0], pair_cols[0] + 7))
        assert all(cols[r * n_kpt + k] == cols[r * n_kpt + k + 1] for r in range(7))   # the two keypoints of a pair share columns
    assert lib.kpn_debug_kmap(0, 20, 4, kmap, None, None) != 0   # unsupported keypoint count
