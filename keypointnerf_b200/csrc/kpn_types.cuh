// Device-side parameter blocks shared by every kernel of the ray-march path.
// Reference behaviour is cited as /root/reference path:line in the functions that use these.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/kpnerf_b200.h"

namespace kpn {

constexpr int MAXV = KPN_MAX_VIEWS;
constexpr int MAXK = KPN_MAX_KPT;
constexpr int NLAYER = KPN_NUM_LAYERS;
constexpr int MAX_SPL = 4;  // sp_level upper bound

// Channel-last feature atlas of one source map: [V][H][W][C] (C padded as noted).
struct MapDesc {
  const void* ptr;
  int C, H, W;  // C = stored channels per texel
};

// Raw (un-derived) scene scalars/matrices exactly as the caller passed them.
struct RawScene {
  float KRT[MAXV * 16];
  float extrin[MAXV * 16];
  float kpt3d[MAXK * 3];
  float bounds[6];
};

struct RawTarget {
  float K[16];
  float RT[16];
};

// Derived per-scene constants (built on device by prep_scene_kernel, no host sync).
struct DevScene {
  int V, K;
  float wm1, hm1;          // cam width-1, height-1
  float znear, zfar;
  float sdf_invalid;       // 0.1 / nml_scale (reference src/model.py:982)
  int use_fg;
  float P[MAXV][12];       // KRT rows 0..2 (3x4)
  float E[MAXV][12];       // extrin rows 0..2
  float C[MAXV][3];        // source camera centres (inverse(KRT)[:3,3], src/model.py:823-824)
  float kc[MAXV][MAXK][3]; // keypoints in each source camera frame (src/spatial.py:85)
  float bounds[6];         // padded by (-0.01,+0.01) (src/model.py:1193)
  int fgbox[MAXV][4];      // per view [x0, x1, y0, y1]: bounding box of the non-zero foreground texels (x1 < 0: none)
  float sp_scale, inv2sig2;
  int sp_level;
  float freq[MAX_SPL];     // float32(pi * 2^l) (src/spatial.py:41-47)
  MapDesc f64, f8, ftex, img, fg;
};

struct DevTarget {
  float invK[9];           // inverse(K[:3,:3]) (src/model.py:1031)
  float R[9];
  float o[3];              // camera centre -t^T R (src/model.py:1036): the origin of every lattice ray
  float znear, zfar;
  int x0, y0, step, nx, ny;
  int step_y;              // lattice step along y (== step for the reference's square lattices)
  float win[MAXV][4];      // per source view [u_lo, u_hi, v_lo, v_hi]: a sample whose normalised projection lies outside can not be
                           // valid (frustum +-1.01 intersected with the dilated foreground bounding box); conservative
};

// Packed dense layers for the fp32 SIMT engine: Wt [K][ldw] transposed, zero padded to ldw = roundup(N,32).
struct DevWeightsF32 {
  const float* wt[NLAYER];
  const float* bias[NLAYER];
  int K[NLAYER], N[NLAYER], ldw[NLAYER];
  float ani_al_abs;
};

// Where the samples of a shading launch come from.  The grid fields of mode 2 share storage with the pointers, which that mode
// does not read, so that the struct (a kernel parameter of every shading kernel) keeps the layout of modes 0 and 1.
struct SampleSrc {
  int mode;            // 0: rays (p = o(ray) + d(ray)*z(ray, i)),  1: explicit points,  2: grid points (no view direction)
  int S;               // samples per ray (mode 0)
  union {
    struct {
      const float* ray_d;  // (R,3) unit directions
      const float* z;      // (R,S) depths; nullptr: the coarse pass' uniform depths, recomputed from ray_nf (never stored)
      const float* ray_nf; // (R,2) near/far along the ray (used when z == nullptr)
      const float* pts;    // (n,3)   (mode 1)
      const float* view;   // (n,3)   (mode 1)
      const float* o;      // (R,3) ray origins (mode 0)
    };
    struct {
      float g_org[3], g_sp[3];   // grid origin and spacing (mode 2): p[a] = g_org[a] + g_sp[a] * idx_a, no FMA contraction
      int g_nx, g_ny;            // grid extent along x, y (mode 2); point id0 + id is (k g_ny + j) g_nx + i
      long long g_id0;           // grid id of the launch's sample 0 (mode 2)
    };
  };
};
static_assert(sizeof(SampleSrc) == 8 + 6 * sizeof(void*), "the grid fields fit in the pointers' storage");

// Where a shading launch puts its per-sample results.
//   query mode (KeypointNeRF.query, query_mode 1): out5[id] = [sdf_raw, rad, r, g, b], dense by sample id.
//   geometry-only query (query_mode 2): out2[id] = [sdf_raw, rad], dense by sample id; no colour work.
//   render mode: compact records indexed by the sample's position in the work list (list_base + index): ao[pos] = (alpha, sdf),
//   rgb[pos] = blended colour (written only for samples with alpha > 0).  Nothing is stored for invalid samples.
struct ShadeOut {
  union {
    float* out5;   // query mode, else nullptr
    float* out2;   // geometry-only query mode, else nullptr
  };
  float2* ao;      // render mode
  float* rgb;      // render mode, 3 floats per list position
  int list_base;   // absolute list position of this launch's first entry
};

// Segment of a ray's samples handled by one compaction pass of an early-ray-termination render (s_hi == 0: all samples).
struct ErtSegment {
  int s_lo, s_hi;
  const float* ray_alpha;   // accumulated alpha of the earlier segments per ray of the chunk, or nullptr
  float eps;
};

enum Layer {
  L_GEO0 = 0, L_GEO1, L_GEO2, L_GEO3, L_DEN0, L_DEN1, L_DEN2, L_CMP,
  L_RE0, L_RE1, L_BASE0, L_BASE1, L_VIS1A, L_VIS1B, L_VIS2A, L_VIS2B, L_OUT0, L_OUT1, L_OUT2
};

}  // namespace kpn
