"""Host-side checks of two contracts of the tensor-core kernels (keypointnerf_b200/csrc/kpn_shade_tc.cu, kpn_tc.cuh) that a GPU
run would only show as a slowdown or as a subtle numerical drift:

  * the shared-memory activation-tile layout `a_word_off` (row threads store 16-byte runs of their row, 32 consecutive rows per
    warp; the accumulator epilogues store one word per lane from the wgmma fragment): a bijection, and free of bank conflicts on
    both sides;
  * the view pooling identity: mean = S1, var = S2 - S1^2 (2 - sum pw) with S1 = sum pw x, S2 = sum pw x^2 is the reference's
    weighted mean / variance (reference src/utils.py:722-748, restated in oracle/kpnerf_oracle.py) for weights that do NOT sum to 1
    exactly (they are normalised with a 1e-6 guard, reference src/model.py:757-759).
"""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "keypointnerf_b200", "csrc", "kpn_tc.cuh")).read()
SHADE = open(os.path.join(ROOT, "keypointnerf_b200", "csrc", "kpn_shade_tc.cu")).read()


def a_word_off(rows, r, c):
    return (((c >> 2) * (rows >> 3) + (r >> 3)) * 128) + (r & 7) * 16 + (c & 3) * 4


def test_python_restatement_matches_the_source():
    m = re.search(r"a_word_off\(int r, int c\) \{\s*return \(uint32_t\)\((.*?)\);\s*\}", SRC, re.S)
    assert m, "a_word_off not found"
    assert m.group(1).replace(" ", "") == "(((c>>2)*(ROWS>>3)+(r>>3))*128)+(r&7)*16+(c&3)*4"
    # the fragment epilogues address pair m of the accumulator as row 16*wq + lane/4 + 8*(m&1), word 4*(m>>1) + lane%4
    assert "const int r = 16 * wq + (lane >> 2) + 8 * (m & 1), c = 4 * (m >> 1) + (lane & 3);" in SHADE


def test_staging_words_are_a_bijection_per_word():
    for rows, words in ((64, 120), (128, 56)):
        idx = {a_word_off(rows, r, c) for r in range(rows) for c in range(words)}
        assert len(idx) == rows * words and max(idx) == rows * words * 4 - 4 and all(i % 4 == 0 for i in idx)


def test_no_bank_conflicts_on_either_side():
    for rows in (64, 128):
        # row threads: one 16-byte store per lane of 32 consecutive rows (run start c % 4 == 0), served per quarter warp
        for r0 in range(0, rows, 32):
            for c in range(0, 64, 4):
                for q in range(4):
                    banks = {(a_word_off(rows, r0 + 8 * q + i, c) // 4 + j) % 32 for i in range(8) for j in range(4)}
                    assert len(banks) == 32
    # accumulator epilogue (64-row tiles): one word per lane, pair m of the fragment of row warp wq
    for wq in range(4):
        for m in range(32):
            banks = {(a_word_off(64, 16 * wq + (lane >> 2) + 8 * (m & 1), 4 * (m >> 1) + (lane & 3)) // 4) % 32 for lane in range(32)}
            assert len(banks) == 32


def test_running_sum_pooling_equals_weighted_mean_and_variance():
    rng = np.random.default_rng(0)
    x = rng.standard_normal((1000, 3, 64))
    pw = rng.random((1000, 3, 1))
    pw = pw / (pw.sum(1, keepdims=True) + 1e-6)          # the reference's normalisation: sums to slightly less than 1
    mean = (pw * x).sum(1)
    var = (pw * (x - mean[:, None]) ** 2).sum(1)
    s1 = (pw * x).sum(1)
    s2 = (pw * x * x).sum(1)
    var2 = s2 - s1 * s1 * (2.0 - pw.sum(1))
    np.testing.assert_allclose(s1, mean, rtol=0, atol=0)
    np.testing.assert_allclose(var2, var, rtol=1e-9, atol=1e-12)
