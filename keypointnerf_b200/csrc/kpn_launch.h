// Host-side launcher declarations (implemented next to their kernels).
#pragma once
#include "kpn_types.cuh"
#include "kpn_tc_types.cuh"

namespace kpn {

cudaError_t launch_pack_nhwc_f32(const float* in, float* out, int V, int C, int H, int W, int Cp, cudaStream_t st);
cudaError_t launch_prep_scene(const RawScene* raw, DevScene* sc, cudaStream_t st);
cudaError_t launch_fg_box(DevScene* sc, int n_views, cudaStream_t st);
cudaError_t launch_prep_target(const RawTarget* raw, DevTarget* tg, const DevScene* sc, cudaStream_t st);
// rays of lattice pixels r0 .. r0 + n - 1 of the target: o, d (n,3), near/far before the bounding-box clip (n,2)
cudaError_t launch_camera_rays(const DevTarget* tg, long long r0, long long n, float* o, float* d, float* nf, cudaStream_t st);
// ray_o, ray_d (nr,3): the chunk's rays; nf_in (nr,2): their near/far before the clip (coarse pass, zbuf == nullptr; may alias
// nothing the kernel writes); ray_nf (nr,2): the clipped near/far (written by the coarse pass)
cudaError_t launch_front(const DevScene* sc, const DevTarget* tg, int nr, int S, const float* zbuf, const float* ray_o,
                         const float* ray_d, const float* nf_in, float* ray_nf, int* list, int list_base, int* counter, int* ray_start,
                         int* ray_cnt, const ErtSegment& ert, cudaStream_t st);
cudaError_t launch_compact(const DevScene* sc, const SampleSrc& src, long long n, int* list, int* counter, float* out, int out_w,
                           uint8_t* valid_out, cudaStream_t st);
cudaError_t launch_composite(const int* list, const float2* ao, const float* rgb, const int* start0, const int* cnt0,
                             const int* start1, const int* cnt1, const float* zbuf, const float* ray_nf, int r0, int nr, int S,
                             long long plane, float* color, float* depth, float* alpha, float* sdf, float* ray_alpha, float* cw,
                             cudaStream_t st);
cudaError_t launch_resample(const int* list, const float* cw, const int* start0, const int* cnt0, const int* start1, const int* cnt1,
                            const float* ray_nf, int nr, int Sc, int Sf, float* zout, float* contrib_out, cudaStream_t st);
// One shading batch: the samples of list[0 .. *counter) (device-side count, at most n_max) of src, shaded with the scene sc
// (n_views views, n_kpt keypoints); `so` says where the results go.  Built once per batch (kpn_api.cu) and passed to the engine's
// launcher, which records after_geo (if not null) once the geometry is shaded and adds the kernels it enqueues to *launches.
struct ShadeBatch {
  const DevScene* sc;
  int n_views, n_kpt;
  SampleSrc src;
  const int* list;
  const int* counter;
  long long n_max;
  int query_mode;
  ShadeOut so;
  int num_sms;
  cudaStream_t st;
  const DevWeightsF32* wf32;   // fp32 engine
  // tensor-core engine: geometry front (L0-L3 + pooling) and density tail kernels, then the colour kernel on the samples with
  // density > 0 (query_mode 2: no colour kernel).  n_views: 3 or 4 (tc_supported); wblob: full fp16 W_hi tiles of every stage;
  // wlo: W_lo tiles of stages 4, 5 (tc_weight_lo_bytes); lo_mask: the W_lo and A_lo passes of the density tail (stages 4, 5:
  // bits 4, 5 and 6, 7); lat: n_max x 48 bytes, pool: tc_pool_bytes(n_max), list2: n_max entries, count2: device int (zeroed by
  // the caller).
  const TcConsts* tcc;
  const uint8_t *wblob, *wlo;
  int lo_mask;
  uint4* lat;
  float* pool;
  int2* list2;
  int* count2;
  cudaEvent_t after_geo;
  unsigned long long* launches;
};
cudaError_t launch_shade_simt(const ShadeBatch& b);
// ---- backward of the fp32 engine (kpn_grad.cu) ----
// Where each layer's gradient sits in a packed gradient vector: dW of layer l at wo[l] ((n_out, n_in) row-major, the layout of
// the folded weight), db at bo[l], d ani_al at ani; `total` floats.  The row-major weight copy (launch_weights_rowmajor) uses
// the same offsets wo[l].
struct GradLayout {
  int wo[NLAYER], bo[NLAYER];
  int ani, total;
};
// The composite backward's inputs (dL/d of one pass' per-ray outputs, planes of `plane` rays at ray r0 + i; nullptr = 0) and
// per-list-position outputs: d_ao = (d rad, d sdf_raw), d_rgb (3 floats); at = scratch of one float2 per list position.
struct RayGrad {
  const float *color, *alpha, *depth, *sdf;
};
cudaError_t launch_composite_backward(const int* list, const float2* ao, const float* rgb, const int* start, const int* cnt,
                                      const float* zbuf, const float* ray_nf, int r0, int nr, int S, long long plane, const RayGrad& g,
                                      float2* d_ao, float* d_rgb, float2* at, int num_sms, cudaStream_t st);
// The shading backward of the samples of batch b (b.so.list_base: list position of the batch's first entry): d_ao / d_rgb per
// list position in, every layer's dW / db / d ani_al added into CTA slice `blockIdx.x` of `slices` (b.num_sms slices of
// lay.total floats), the feature-map gradients added (atomics) into d_f64 / d_f8 / d_ftex ([V][H][W][C], the atlases' extents).
struct ShadeGrad {
  const float2* d_ao;
  const float* d_rgb;
  const float* wr;        // row-major copy of every folded weight (launch_weights_rowmajor)
  GradLayout lay;
  float* slices;
  float *d_f64, *d_f8, *d_ftex;
  float ani_sign;         // sign(ani_al): the layers see |ani_al|
};
cudaError_t launch_shade_simt_backward(const ShadeBatch& b, const ShadeGrad& g);
// The work list of one pass rewritten in ray order: start_out = the exclusive scan of cnt (nr rays), ray i's cnt[i] entries copied
// from list_in[start_in[i] ..] to list_out[start_out[i] ..].  scan_tmp holds canonical_list_temp_bytes(nr) bytes.
size_t canonical_list_temp_bytes(int nr);
cudaError_t launch_canonical_list(const int* list_in, const int* start_in, const int* cnt, int nr, int* list_out, int* start_out,
                                  void* scan_tmp, size_t scan_bytes, int num_sms, cudaStream_t st);
cudaError_t launch_weights_rowmajor(const DevWeightsF32* w, float* wr, const GradLayout& lay, cudaStream_t st);
// out[i] = sum over the n slices, in slice order, of slices[s * total + i]
cudaError_t launch_grad_reduce(const float* slices, int n, int total, float* out, cudaStream_t st);
cudaError_t launch_shade_tc(const ShadeBatch& b);
cudaError_t launch_shade_tc_v4(const ShadeBatch& b);   // the 4-view instantiation (kpn_shade_tc_v4.cu)
size_t tc_pool_bytes(long long n_max);
// Device watchdog words of the tensor-core kernels: TC_WD_WORDS per module, one module per view-count translation unit.
constexpr int TC_WD_WORDS = 8;
constexpr int TC_WD_MODULES = 2;
cudaError_t tc_watchdog_words(void* w[TC_WD_MODULES]);   // device address of every module's words
cudaError_t tc_watchdog_addr_v4(void** p);   // device address of the 4-view module's words
size_t tc_weight_blob_bytes(int n_kpt);
size_t tc_weight_lo_bytes(int n_kpt);
bool tc_supported(int n_views, int n_kpt, int sp_level);
// source-view decode (kpn_decode.cu): cams = V x {double ir[9], fx, fy, cx, cy, k1, k2, p1, p2, k3} on the device
cudaError_t launch_decode_views(const uint8_t* images, const uint8_t* masks, const void* cams, int V, int H0, int W0, int factor,
                                float* out_img, uint8_t* out_mask, cudaStream_t st);
// marching cubes (kpn_mesh.cu) over f[nz][ny][nx], nx * ny * nz <= INT32_MAX.  classify: vcnt (per point) and tcnt (per cell)
// become the exclusive scans vofs / tofs, cases[cell] the case byte, totals[2] (device) = [vertices, faces]; scan_tmp holds
// mc_scan_temp_bytes(nx * ny * nz) bytes.  emit: vertices / normals (may be nullptr) / faces at those offsets.
size_t mc_scan_temp_bytes(int n);
cudaError_t launch_mc_classify(const float* f, int nx, int ny, int nz, float level, unsigned int* vcnt, uint8_t* cases, unsigned int* tcnt,
                               unsigned long long* totals, void* scan_tmp, size_t scan_bytes, cudaStream_t st);
cudaError_t launch_mc_emit(const float* f, int nx, int ny, int nz, float level, const float origin[3], const float spacing[3],
                           const unsigned int* vofs, const uint8_t* cases, const unsigned int* tofs, float* verts, float* normals,
                           int* faces, long long n_faces, cudaStream_t st);
int max_coarse_samples();
int simt_max_kpt();
int simt_max_geo_input();   // widest geometry-layer-0 input ((1 + 2 sp_level) n_kpt + 64) the fp32 engine's tile rows hold

}  // namespace kpn
