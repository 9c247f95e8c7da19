"""Golden vectors for keypoint counts other than 18 and 24, from the UNMODIFIED reference on CPU (same harness and file format
as make_golden.py, whose functions this reuses).

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_kpt.py            # every case below
    python tests/golden/make_golden_kpt.py tiny_k5    # only the named cases
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402

_c = G._c
# few keypoints (the first row thread of the geometry front kernel builds no keypoint pair), an odd count, the first count
# above 24 (non-square, level 2 with offsets), the maximum count of 32 (one warpgroup per front CTA), and 32 keypoints at the
# size of BASELINE config 2 (one strided pass of the 512x512x128 frame, hull scene)
KPT_CASES = {
    "tiny_k5": _c(src_size=64, tgt_size=32, zoom=2.0, azimuth=0.5, level=1, S_c=12, S_f=8, fine=True, n_kpt=5,
                  scene_seed=6, w_seed=11, capture="all"),
    "tiny_k17": _c(src_size=64, tgt_size=32, zoom=2.0, level=1, S_c=12, S_f=8, fine=True, n_kpt=17, scene_seed=7,
                   capture="all"),
    "rect_k25": _c(src_size=128, src_height=80, tgt_size=48, tgt_width=48, tgt_height=32, zoom=3.0, azimuth=2.5, level=2,
                   x_off=1, y_off=1, S_c=12, S_f=8, fine=True, n_kpt=25, scene_seed=3, w_seed=5, capture="all"),
    "tiny_k32": _c(src_size=64, tgt_size=32, zoom=2.0, azimuth=1.5, level=1, S_c=12, S_f=8, fine=True, n_kpt=32,
                   scene_seed=5, w_seed=9, capture="all"),
    "cfg2_pass_k32": _c(x_off=3, y_off=5, S_c=128, n_kpt=32, capture="some"),
}

if __name__ == "__main__":
    G.CASES.update(KPT_CASES)
    if len(sys.argv) == 1:
        sys.argv += list(KPT_CASES)
    G.main()
