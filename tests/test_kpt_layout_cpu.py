"""Tensor-core weight packing for every keypoint count the engine covers (1..32), host code only (no GPU): the K index each
input of a geometry stage is multiplied with (kpn_debug_kmap), and the layer-0 layout the front kernel's two row threads write."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__ as G
from keypointnerf_b200 import _lib as L

COUNTS = list(range(1, 33))


@pytest.fixture(scope="module")
def lib():
    G.build()
    return L.load()


def kmap(lib, stage, n_kpt, n):
    out = (C.c_int * n)()
    kbias, kpad = C.c_int(), C.c_int()
    assert lib.kpn_debug_kmap(stage, n_kpt, n, out, C.byref(kbias), C.byref(kpad)) == 0
    return np.array(out), kbias.value, kpad.value


def n_inputs(stage, n_kpt):
    return {0: 7 * n_kpt + 64, 1: 128, 2: 136, 3: 120, 4: 128, 5: 64}[stage]


def layer0_runs(km, kbias, kpad, n_kpt):
    """Recover the run split (pairs PA, channels FA of the first thread) from the map and check that every fp16 word holds what
    the kernel writes there: [pairs 0..PA-1 | channels 0..FA-1 | pairs PA..NP-1 | channels FA..63 | bias | zero padding], where
    word 7 j + r of a pair holds encoding element r of keypoints 2 j (low half) and 2 j + 1 (high half)."""
    n_pair = (n_kpt + 1) // 2
    enc, feat = km[:7 * n_kpt], km[7 * n_kpt:]
    pair_word = np.array([enc[k] // 2 for k in range(0, n_kpt, 2)])   # word of element r = 0 of each pair
    pa = int(np.sum(pair_word < feat[0] // 2)) if len(feat) else n_pair
    fa = int(np.sum(feat // 2 < (pair_word[pa] if pa < n_pair else kbias // 2)))
    c1 = 7 * pa + fa // 2
    want = []
    for j in range(n_pair):
        base = 7 * j if j < pa else c1 + 7 * (j - pa)
        want += [(r, k, 2 * (base + r) + (k & 1)) for r in range(7) for k in (2 * j, 2 * j + 1) if k < n_kpt]
    got = [(r, k, int(enc[r * n_kpt + k])) for r, k, _ in want]
    assert got == want
    tail0 = c1 + 7 * (n_pair - pa)
    assert list(feat) == [14 * pa + c if c < fa else 2 * tail0 + (c - fa) for c in range(64)]
    assert kbias == 2 * (tail0 + (64 - fa) // 2)
    return pa, fa, c1


@pytest.mark.parametrize("n_kpt", COUNTS)
def test_weight_packing_is_a_bijection_for_every_count(lib, n_kpt):
    """Every input of every geometry stage is multiplied with its own K index, the bias row has a K index of its own, and
    everything fits the padded K, a multiple of 16.  Counts outside 1..32, stages past 5 and an input count other than the
    stage's own are refused."""
    for stage in range(6):
        n = n_inputs(stage, n_kpt)
        ks, kbias, kpad = kmap(lib, stage, n_kpt, n)
        assert len(set(ks.tolist())) == n and kbias not in ks
        assert 0 <= ks.min() and max(ks.max(), kbias) < kpad and kpad % 16 == 0
        buf = (C.c_int * (n + 1))()
        assert lib.kpn_debug_kmap(stage, n_kpt, n + 1, buf, None, None) != 0
        assert lib.kpn_debug_kmap(stage, n_kpt, n - 1, buf, None, None) != 0
    for bad in (0, 33, -1):
        buf = (C.c_int * max(7 * bad + 64, 1))()
        assert lib.kpn_debug_kmap(0, bad, 7 * bad + 64, buf, None, None) != 0
    buf = (C.c_int * 64)()
    assert lib.kpn_debug_kmap(6, n_kpt, 64, buf, None, None) != 0


def front_writers(pa, fa, c1, kpad, n_kpt):
    """The words of a layer-0 row that each writer of geo_front_kernel stores, restated from the kernel: row thread h = 0 its
    pairs' encodings (a_put_span<0, 7 PA>), row thread h = 1 its pairs' encodings (a_put_span<C1, NE>) and the bias column with
    the K padding after the feat64 channels FA..63 (a_put_span<C1 + NE + NF, K0P / 2 - C1 - NE - NF>), and gather_feat64 the two
    words of each float4 group c4 of feat64 channels at column 7 PA + 2 c4 (c4 < FA / 4) or C1 + NE + 2 (c4 - FA / 4)."""
    ne, nf = 7 * ((n_kpt + 1) // 2 - pa), (64 - fa) // 2
    w = {"h0 encodings": range(0, 7 * pa), "h1 encodings": range(c1, c1 + ne),
         "h1 bias / padding": range(c1 + ne + nf, kpad // 2)}
    for c4 in range(16):
        col = 7 * pa + 2 * c4 if 4 * c4 < fa else c1 + ne + 2 * (c4 - fa // 4)
        w[f"feat64 group {c4}"] = range(col, col + 2)
    return w


def assert_partition(writers, n_words):
    """Every word of [0, n_words) is stored by exactly one writer, and no writer stores outside it."""
    who = [[] for _ in range(n_words)]
    for name, words in writers.items():
        for c in words:
            assert 0 <= c < n_words, f"{name} stores word {c}, outside [0, {n_words})"
            who[c].append(name)
    wrong = {c: names for c, names in enumerate(who) if len(names) != 1}
    assert not wrong, f"words not stored exactly once: {wrong}"


@pytest.mark.parametrize("n_kpt", COUNTS)
def test_layer0_runs_are_chunk_aligned(lib, n_kpt):
    """The two row threads of the front kernel write one contiguous run of 32-bit words each, with 16-byte stores: both runs
    start on a 4-word chunk and both have a whole number of chunks; the first thread gathers whole float4 groups of feat64.
    The L3 rows of a tile are staged over its activation tile, so every word of the next tile's layer-0 input must be stored
    again: the front kernel's writers cover the row exactly once, each feat64 word at the column the weights expect, and the
    same holds for words 64..71 of the layer-1 and layer-2 inputs (after the epilogue's words 0..63)."""
    km, kbias, kpad = kmap(lib, 0, n_kpt, n_inputs(0, n_kpt))
    pa, fa, c1 = layer0_runs(km, kbias, kpad, n_kpt)
    assert pa % 2 == 0 and fa % 4 == 0 and 0 < c1 < kpad // 2
    assert c1 % 4 == 0 and (kpad // 2 - c1) % 4 == 0
    writers = front_writers(pa, fa, c1, kpad, n_kpt)
    assert_partition(writers, kpad // 2)
    feat = km[7 * n_kpt:]
    for c in range(64):   # float4 group c // 4 packs channels (4g, 4g + 1) in its first word, (4g + 2, 4g + 3) in its second
        assert feat[c] == 2 * writers[f"feat64 group {c // 4}"][(c % 4) // 2] + c % 2, c
    assert kbias == 2 * writers["h1 bias / padding"][0]   # the H2_ONE word: 1.0 in the low half
    # layer 1: the epilogue's words 0..63, the bias chunk of thread h = 0 (a_put<64, 8>)
    k1, kb1, kp1 = kmap(lib, 1, n_kpt, n_inputs(1, n_kpt))
    assert_partition({"epilogue": range(0, 64), "h0 bias chunk": range(64, 72)}, kp1 // 2)
    assert k1.tolist() == list(range(128)) and kb1 == 128
    # layer 2: the epilogue's words 0..63, feat8 channels 0..3 from thread h = 0 (a_put_span<64, 2>), channels 4..7, the bias
    # column and the padding from thread h = 1 (a_put_span<66, 6>)
    k2, kb2, kp2 = kmap(lib, 2, n_kpt, n_inputs(2, n_kpt))
    assert_partition({"epilogue": range(0, 64), "h0 feat8": range(64, 66), "h1 feat8 / bias / padding": range(66, 72)}, kp2 // 2)
    assert k2.tolist() == list(range(136)) and kb2 == 2 * 68
    # an odd count's last pair has one unused slot: nothing maps to the high half of its words
    if n_kpt % 2:
        j = n_kpt // 2
        assert not (set(2 * (km[r * n_kpt + 2 * j] // 2) + 1 for r in range(7)) & set(km.tolist()))
    # padded K: the bias column plus the pairs rounded up to a multiple of 16 fp16 elements
    assert kpad == (14 * ((n_kpt + 1) // 2) + 65 + 15) // 16 * 16


@pytest.mark.parametrize("n_kpt", [18, 24])
def test_layer0_layout_of_18_and_24_is_unchanged(lib, n_kpt):
    """18 and 24 keypoints keep the layout they have always had (4 pairs + feat64 channels 0..39 in the first thread's run):
    another split would reorder layer 0's K sum and change the last bits of every output."""
    pa, fa, n_pair = 4, 40, n_kpt // 2

    def old(i):
        if i < 7 * n_kpt:
            r, k = divmod(i, n_kpt)
            j = k // 2
            col = 7 * j + r if j < pa else 7 * pa + fa // 2 + 7 * (j - pa) + r
            return 2 * col + (k & 1)
        c = i - 7 * n_kpt
        return 14 * pa + c if c < fa else 2 * (7 * pa + fa // 2 + 7 * (n_pair - pa)) + (c - fa)

    km, kbias, kpad = kmap(lib, 0, n_kpt, n_inputs(0, n_kpt))
    assert km.tolist() == [old(i) for i in range(7 * n_kpt + 64)]
    assert kbias == 2 * (7 * n_pair + 32) and kpad == {18: 192, 24: 240}[n_kpt]
