/*
 * kpnerf_b200 -- C ABI of the CUDA-native (H100, sm_90a) KeypointNeRF ray-march hot path.
 *
 * The reference (facebookresearch/KeypointNeRF) has no FFI: its seam for this path is
 * the Python method surface of class KeypointNeRF (SURVEY.md section 8b).  Each entry
 * point below names the reference interface it stands in for; the Python shim
 * keypointnerf_b200/model.py binds them with ctypes and exposes the reference's own
 * method names and argument meaning.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch types.  Every pointer argument is either a
 *     HOST pointer or a DEVICE pointer according to the `mem` field/argument next to it.
 *     With KPN_MEM_HOST the library performs the host<->device copies itself on `stream`
 *     (asynchronously when the host memory is pinned).
 *   - all float tensors are fp32, dense, row-major, with the layouts of the reference's
 *     torch tensors (NCHW feature maps, (V,4,4) cameras ...).
 *   - every call is enqueued on the caller's CUDA stream (`stream` = cudaStream_t cast to
 *     void*, NULL = legacy default stream); no call synchronises the device, except
 *     kpn_set_weights (host-side packing, once per checkpoint) and calls that take
 *     pageable host memory (cudaMemcpyAsync semantics).
 *   - return value: KPN_OK or a negative kpn_status; kpn_last_error() gives the text.
 *     There is no CPU fallback: without a CUDA device kpn_create fails.
 */
#ifndef KPNERF_B200_H
#define KPNERF_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KPN_ABI_VERSION 5
#define KPN_MAX_VIEWS 4
#define KPN_MAX_KPT 32
#define KPN_NUM_LAYERS 19

typedef enum {
  KPN_OK = 0,
  KPN_ERR_ARG = -1,         /* bad argument / unsupported shape (reference: Python assert) */
  KPN_ERR_CUDA = -2,        /* CUDA runtime error */
  KPN_ERR_STATE = -3,       /* weights or scene not set */
  KPN_ERR_UNSUPPORTED = -4  /* reference: NotImplementedError */
} kpn_status;

typedef enum { KPN_MEM_DEVICE = 0, KPN_MEM_HOST = 1 } kpn_mem;

typedef struct kpn_ctx kpn_ctx;

/* One dense layer exactly as it sits in the reference state_dict (HOST pointers).
 * weight-normed layer (reference src/utils.py:542-543): w = weight_v (out,in), g = weight_g (out,1);
 * plain layer: w = weight (out,in), g = NULL. */
typedef struct {
  const float* w;
  const float* g;
  const float* bias;
  int n_out, n_in;
} kpn_layer;

/* Layer order (reference parameter names, SURVEY.md Appendix D):
 *  0..3  mlp_geo.layers1.layers.{0..3}.linear     4..6  mlp_geo.layers2.layers.{0..2}.linear
 *  7     ibr_compress_gfeat                        8,9   mlp_tex.ray_encoder.{0,2}
 *  10,11 mlp_tex.base_layer.{0,2}                  12,13 mlp_tex.vis_layer1.{0,2}
 *  14,15 mlp_tex.vis_layer2.{0,2}                  16..18 mlp_tex.out_layer.{0,2,4} */
typedef struct {
  kpn_layer layer[KPN_NUM_LAYERS];
  float ani_al;      /* mlp_tex.ani_al (reference src/model.py:1245) */
  int n_kpt;         /* sp_args.n_kpt */
  int sp_level;      /* sp_args.sp_level (3) */
  float sp_scale;    /* sp_args.scale */
  float sp_sigma;    /* sp_args.sigma */
} kpn_weights;

/* Source-side inputs of KeypointNeRF.query (reference src/model.py:690-782): cam dict,
 * sp_data, cached feature maps, source images and foreground masks. */
typedef struct {
  int n_views, n_kpt;            /* 1 <= n_views <= KPN_MAX_VIEWS (engine 0 / 2-4: 3 or 4 views; engine 1: any) */
  float src_width, src_height;   /* cam["width"], cam["height"] */
  float znear, zfar;             /* cam["znear"], cam["zfar"] */
  float nml_scale;               /* cam["nml_scale"] */
  const float* KRT;              /* (V,4,4) */
  const float* extrin;           /* (V,4,4) sp_data["extrin"] */
  const float* kpt3d;            /* (K,3)   sp_data["kpt3d"][0] */
  const float* bounds;           /* (2,3)   config["bounds"][0] */
  const float* feat64;  int f64_c, f64_h, f64_w;     /* feat_geo[0] (V,C,H,W) */
  const float* feat8;   int f8_c, f8_h, f8_w;        /* feat_geo[1] */
  const float* feat_tex; int ftex_c, ftex_h, ftex_w; /* feat_tex */
  const float* img;     int img_h, img_w;            /* img_in (V,3,H,W) */
  const uint8_t* fg;    int fg_h, fg_w;              /* src_foreground_mask (V,1,H,W) bool; NULL = disable_fg_mask */
  int mem;                                           /* kpn_mem of ALL pointers above */
  int layout;                                        /* bit mask of KPN_NHWC_*: that map is already stored [V][H][W][C]
                                                        (what the channels-last encoders emit): no re-layout pass; a DEVICE
                                                        map is then gathered from IN PLACE and must stay alive and unchanged
                                                        until the next kpn_set_scene */
} kpn_scene;
#define KPN_NHWC_FEAT64 1
#define KPN_NHWC_FEAT8 2
#define KPN_NHWC_FEATTEX 4

/* Target camera + pixel lattice (reference src/model.py:973-976,1018-1036).
 * Pixel (i,j), 0<=i<nx, 0<=j<ny is x = x0 + step*i, y = y0 + step_y*j; outputs are indexed [j*nx+i].
 * The reference's strided pass (level, stride=[x_off,y_off]) is step=step_y=2^(level-1), x0=x_off, y0=y_off,
 * nx=width/step, ny=height/step; a full frame is step=1, nx=width, ny=height.  step_y = 0 means step_y = step; a
 * different step_y gives the rectangular lattice phases of the multi-GPU frame partition (one phase per rank: every
 * phase sees the whole image, so the ranks are load-balanced by construction; reference src/model.py:916-923). */
typedef struct {
  const float* K;    /* (4,4) cam_tar["K"][0] */
  const float* RT;   /* (4,4) cam_tar["RT"][0] */
  float znear, zfar;
  int x0, y0, step, nx, ny;
  int mem;           /* kpn_mem of K, RT */
  int step_y;        /* 0: same as step */
} kpn_target;

typedef struct {
  int sample_per_ray_c;   /* config["sample_per_ray_c"] */
  int sample_per_ray_f;   /* config["sample_per_ray_f"] */
  int fine;               /* config["fine"] */
  float ert_eps;          /* early-ray-termination transmittance threshold; 0 = off (reference behaviour) */
  const float* z_fine_override; /* optional (R, S_c+S_f) sorted depths replacing the resampled ones (test hook; same kpn_mem as kpn_out) */
  int engine;             /* 0 = default: tensor cores (wgmma), fp16 operands, fp32 accumulate; the density tail (stages P0|compress,
                                 P1) runs with two-term (hi+lo) weights and activations;
                             1 = fp32 CUDA-core engine (parity anchor, ~25x slower; the ONLY engine for shapes the tensor-core
                                 engine does not cover: n_views 1 or 2, sp_level != 3 -- such shapes fail with
                                 KPN_ERR_UNSUPPORTED unless engine = 1 is requested explicitly).  Every engine takes any
                                 1 <= n_kpt <= KPN_MAX_KPT;
                             2 = as 0 with single-term fp16 weights in the density tail (more rounding error);
                             3, 4 = as 0 (they selected between two geometry kernels of an earlier architecture; one kernel
                                 serves both here) */
} kpn_opts;

/* An explicit batch of n rays (kpn_render_rays): any pixel subset, camera model or set of cameras.  Ray i marches the points
 * origins[i] + z * dirs[i] for z in [near, far], where [near, far] is near_far[i] tightened to the scene's bounding box exactly as
 * the lattice rays' are (reference src/model.py:1039-1043, 1178-1237, with the ray's own origin); dirs[i] is also the view
 * direction of its samples. */
typedef struct {
  const float* origins;   /* (n,3) ray origins */
  const float* dirs;      /* (n,3) unit directions, used as given (the library does not renormalise) */
  const float* near_far;  /* (n,2) near/far distances along dirs BEFORE the bounding-box clip */
  long long n;
  int mem;                /* kpn_mem of the three arrays */
} kpn_rays;

/* Outputs of batch_render_pifu_nerf (reference src/model.py:1065-1096); any pointer may be NULL. */
typedef struct {
  float* tex_fg;       /* (3,ny,nx) */
  float* depth;        /* (ny,nx) */
  float* alpha;        /* (ny,nx) */
  float* tex_fg_fine;  /* (3,ny,nx) */
  float* depth_fine;   /* (ny,nx) */
  float* alpha_fine;   /* (ny,nx) */
  float* sdf;          /* (ny,nx) */
  float* z_fine;       /* (ny*nx, S_c+S_f) debug: the sorted depths of the fine pass */
  float* contrib;      /* (ny*nx, S_c)     debug: coarse compositing weights */
  int mem;             /* kpn_mem of the pointers above */
} kpn_out;

/* A regular grid of points: point (i,j,k), 0<=i<nx, 0<=j<ny, 0<=k<nz, has id (k*ny + j)*nx + i (x fastest) and position
 * p[a] = origin[a] + spacing[a]*idx_a, computed in fp32 as one multiply then one add (no fused multiply-add), so that a
 * caller can rebuild the points bit for bit. */
typedef struct {
  float origin[3];
  float spacing[3];
  int nx, ny, nz;
} kpn_grid;

typedef struct {
  uint64_t samples_total;   /* samples generated by the last render/query */
  uint64_t samples_valid;   /* samples that passed the validity test and were shaded */
  uint64_t kernel_launches; /* kernels launched by this context since creation */
  uint64_t shade_launches;  /* launches of the dominant (shading) kernel timed since the last kpn_get_stats */
  double shade_ms;          /* their summed device time (CUDA events on the launch stream); 0 unless profiling */
  uint64_t samples_coloured;/* valid samples with density > 0, i.e. shaded by the colour kernel too (tensor-core engine) */
  double geo_ms;            /* the geometry kernel's part of shade_ms (tensor-core engine, profiling on) */
} kpn_stats;

int kpn_abi_version(void);

/* Context = one device's packed weights, packed feature atlases and workspace.
 * Stands in for constructing KeypointNeRF(cfg).cuda() (reference src/model.py:559). */
int kpn_create(int device, kpn_ctx** out);
void kpn_destroy(kpn_ctx* ctx);
const char* kpn_last_error(const kpn_ctx* ctx);

/* Folds weight norm, transposes/pads and uploads the hot-path parameters.
 * Stands in for load_state_dict on mlp_geo / mlp_tex / ibr_compress_gfeat (reference src/model.py:113-117).
 * With a scene bound, new weights with the same n_kpt keep it bound and rewrite its encoding constants (sp_level,
 * sp_scale, sp_sigma), so the next render equals one after a fresh kpn_set_scene; a different n_kpt unbinds it, and
 * kpn_render / kpn_query return KPN_ERR_STATE until kpn_set_scene is called again. */
int kpn_set_weights(kpn_ctx* ctx, const kpn_weights* w);

/* Re-layouts the source feature maps into channel-last atlases and derives per-view constants.  The keypoint-encoding
 * constants come from the weights set last (see kpn_set_weights).
 * Stands in for attach_im_feat / the feat_geo, feat_tex, cam_in, sp_data arguments (reference src/model.py:642-680,922). */
int kpn_set_scene(kpn_ctx* ctx, const kpn_scene* scene, void* stream);

/* KeypointNeRF.batch_render_pifu_nerf, eval branch (reference src/model.py:942-1108);
 * with step=1 it renders what render_pifu_nerf assembles from stride^2 passes (src/model.py:897-940).
 * A lattice of more than 2^31 - 1 rays (nx*ny) is refused with KPN_ERR_ARG, as is a kpn_render_rays batch of more. */
int kpn_render(kpn_ctx* ctx, const kpn_target* target, const kpn_opts* opts, const kpn_out* out, void* stream);

/* The eval branch of batch_render_pifu_nerf (reference src/model.py:1038-1096) on the explicit rays of `rays` instead of a
 * target's pixel lattice: the same coarse pass, fine pass, opts and debug outputs as kpn_render, with the kpn_out planes
 * shaped as a lattice of nx = n, ny = 1 (tex_fg (3,n), depth / alpha / sdf (n), contrib (n,S_c), z_fine and
 * z_fine_override (n,S_c+S_f)).  kpn_render_rays(kpn_camera_rays(T)[idx]) equals kpn_render(T) at the pixels idx bit for bit,
 * for any subset, order or concatenation of cameras.  n == 0: KPN_OK, nothing is done; null arrays or n < 0: KPN_ERR_ARG;
 * no scene: KPN_ERR_STATE; sample counts, engines and their refusals as kpn_render. */
int kpn_render_rays(kpn_ctx* ctx, const kpn_rays* rays, const kpn_opts* opts, const kpn_out* out, void* stream);

/* Gradients of kpn_render_rays (every output a layer of the reference's hot path, mlp_tex.ani_al or a gathered feature map
 * depends on), with the reference's autograd semantics (src/model.py:978-1096, 1150-1176, eval branch, uniform=True).  The
 * ray batch is in the layout of kpn_render_rays; dW of layer l is (n_out, n_in) of the FOLDED weight (g * v / ||v|| for a
 * weight-normed layer), the feature-map gradients are channel-last (V, H, W, C) with the extents of kpn_scene's maps. */
typedef struct {
  float* dW[KPN_NUM_LAYERS];
  float* db[KPN_NUM_LAYERS];
  float* d_ani_al;     /* (1) */
  float* d_feat64;     /* (V, H, W, 64) feat_geo[0] */
  float* d_feat8;      /* (V, H, W, 8)  feat_geo[1] */
  float* d_feat_tex;   /* (V, H, W, 8)  feat_tex */
  int mem;             /* kpn_mem of the pointers above */
} kpn_grads;

/* The backward of kpn_render_rays: grad_out holds dL/d of each output plane of kpn_out (same shapes; NULL plane = zero; z_fine
 * and contrib are ignored), every array of grads is overwritten with dL/d that parameter.  The depths of the fine pass are
 * constants (the reference resamples under torch.no_grad); source images, cameras, keypoints, bounds, rays and masks are data.
 * The forward is recomputed with the fp32 engine whatever opts->engine says, and the gradients are fp32 (CUDA cores); the
 * fine pass uses opts->z_fine_override when set (kpn_mem of grad_out).  Chunking as kpn_render_rays; n == 0 writes zeros.
 * Null arrays, bad sample counts: KPN_ERR_ARG; no weights or scene: KPN_ERR_STATE; ert_eps > 0: KPN_ERR_UNSUPPORTED (the
 * samples early-ray termination skips have gradients). */
int kpn_render_rays_backward(kpn_ctx* ctx, const kpn_rays* rays, const kpn_opts* opts, const kpn_out* grad_out, const kpn_grads* grads,
                             void* stream);

/* The rays kpn_render marches for the target's pixel lattice, pixel j*nx+i at index j*nx+i: origins (R,3) = -t^T R,
 * dirs (R,3) = normalize(K^-1 [x,y,1] R), near_far (R,2) = |znear K^-1 [x,y,1]|, |zfar K^-1 [x,y,1]| (before the bounding-box
 * clip), R = nx*ny.  Needs neither weights nor a scene.  `mem` = kpn_mem of the three outputs (the target's own mem field
 * describes K and RT). */
int kpn_camera_rays(kpn_ctx* ctx, const kpn_target* target, float* origins, float* dirs, float* near_far, int mem, void* stream);

/* KeypointNeRF.query (reference src/model.py:690-782): pts, view (n,3) -> out5 (n,5) = [sdf_raw, rad, r, g, b],
 * valid (n) in {0,1}.  Rows with valid==0 carry out5 = [0,0,0,0,0] (the reference's values there are
 * multiplied by a zero mask downstream, src/model.py:982,996). */
int kpn_query(kpn_ctx* ctx, const float* pts, const float* view, int n, float* out5, uint8_t* valid,
              int mem, const kpn_opts* opts, void* stream);

/* The density field of KeypointNeRF.query on a grid, without the colour branch: out2 (n,2) = [sdf_raw, rad] and valid (n)
 * in {0,1}, n = nx*ny*nz, indexed by grid id.  No per-point input.  A point's [sdf_raw, rad, valid] is bit-identical to
 * columns 0-1 of kpn_query at the same point with the same engine (the view direction only enters the colour).  Rows with
 * valid==0 carry [0,0].  Same engines and shapes as kpn_query; n <= 2^31-1, every extent >= 1, spacing finite and > 0
 * (else KPN_ERR_ARG).  kpn_get_stats reports samples_total = n, samples_valid, and samples_coloured = 0.
 * `mem` = kpn_mem of out2 and valid (valid may be NULL). */
int kpn_query_grid(kpn_ctx* ctx, const kpn_grid* grid, float* out2, uint8_t* valid, int mem, const kpn_opts* opts, void* stream);

/* Marching cubes, first half: classifies the cells of the fp32 volume `field` (DEVICE pointer, f[nz][ny][nx], x fastest)
 * against `level` and scans the per-point vertex and per-cell face counts; writes [n_vertices, n_faces] to counts (host).
 * A corner is inside when f > level (NaN: outside); each grid edge with one inside endpoint gets one vertex.  The workspace
 * (about 9 bytes per point) is kept in the context for kpn_mesh_emit.  More than 2^31-1 points, vertices or faces:
 * KPN_ERR_ARG.  Synchronises `stream` (the counts are needed to size the outputs). */
int kpn_mesh_begin(kpn_ctx* ctx, const float* field, int nx, int ny, int nz, float level, long long counts[2], void* stream);

/* Marching cubes, second half: the mesh of the field passed to the last kpn_mesh_begin (the same pointer, unchanged since;
 * otherwise KPN_ERR_STATE), on the grid origin / spacing (host arrays, as kpn_grid):
 *   vertices (n_vertices,3): one per crossing edge, ordered by (linear index of the edge's lower endpoint a, axis x<y<z), at
 *     p_a + t*(p_b - p_a) with t = (level - f_a)/(f_b - f_a) (an edge with a non-finite t gets its midpoint);
 *   normals (n_vertices,3) or NULL: -grad f / |grad f| interpolated by t between the endpoints' gradients (central
 *     differences inside the grid, one-sided at its border); a zero gradient, or one that a NaN or infinite sample enters,
 *     gives (0,0,0);
 *   faces (n_faces,3) int32 vertex indices, by cell linear index then case-table order, counter-clockwise seen from the side
 *     where f <= level.  Closed and edge-manifold when f <= level on the grid boundary.
 * `mem` = kpn_mem of vertices, normals, faces (which may be NULL when their count is 0). */
int kpn_mesh_emit(kpn_ctx* ctx, const float* field, const float origin[3], const float spacing[3], float* vertices, float* normals,
                  int* faces, int mem, void* stream);

/* Counters of the last call (+ the shading-kernel timings accumulated since the previous
 * kpn_get_stats when profiling is on).  Synchronises `stream` (debug/bench only). */
int kpn_get_stats(kpn_ctx* ctx, kpn_stats* stats, void* stream);

/* Non-blocking health check.  Every render/query enqueues a copy of the tensor-core kernels' device watchdog words into
 * pinned host memory; this call (and the start of every other call) looks at the last copy that has landed.  If a barrier
 * wait gave up (a protocol bug: the affected launch and every later tensor-core launch produced garbage) it returns
 * KPN_ERR_CUDA with the location in kpn_last_error, clears the device flag (re-arming the engine) and the host copy.
 * Callers that synchronise the stream anyway (host outputs) call it right after: RayMarcher.render does. */
int kpn_check_health(kpn_ctx* ctx, void* stream);

/* Pre-sizes every workspace buffer for renders of up to max_rays rays x max_samples samples per ray (coarse + fine), so that
 * later kpn_render calls of at most that size never allocate or free device memory.  Without it buffers grow on demand
 * (cudaFree + cudaMalloc: implicit device synchronisation) the first time a larger size is seen. */
int kpn_reserve(kpn_ctx* ctx, long long max_rays, int max_samples);

/* Source-view decode on the device: what ZJUDataset.__getitem__ does to every view on CPU workers (reference
 * src/zju_dataset.py:266-287): cv2.undistort of the image (float32 / 255) and of the mask, cv2.resize by 1 / factor (INTER_AREA /
 * INTER_NEAREST; factor >= 1 integer, source size divisible by it), image[mask == 0] = 0.  Bit-identical to the cv2 calls.
 *   images (V, H0, W0, 3) uint8 RGB, masks (V, H0, W0) uint8 (non-zero = foreground) or NULL,
 *   cams   (V, 18) double per view: the 9 entries of inverse(K) row-major, then fx, fy, cx, cy, k1, k2, p1, p2, k3,
 *   out_img (V, 3, H0/factor, W0/factor) fp32 in [0, 1], out_mask (V, 1, H0/factor, W0/factor) uint8 in {0, 1} or NULL.
 * `mem` = kpn_mem of every pointer (host pointers are staged through the context's buffers on `stream`). */
int kpn_decode_views(kpn_ctx* ctx, const uint8_t* images, const uint8_t* masks, const double* cams, int n_views, int src_h, int src_w,
                     int factor, float* out_img, uint8_t* out_mask, int mem, void* stream);

/* Debug: the device watchdog words of the tensor-core kernels.  Every barrier wait of those kernels gives up after ~2^20
 * suspended polls instead of hanging the GPU; out16 (host, may be NULL) receives [0] flag (!= 0: some wait gave up; results of
 * that launch are invalid), [1] block, [2] thread, [3] tag of the wait, [4] parity; [5..15] zero.  enable != 0 clears the
 * flag afterwards.  kpn_get_stats reports a raised flag as KPN_ERR_CUDA.  Synchronises the device. */
int kpn_debug_timing(kpn_ctx* ctx, int enable, unsigned long long* out16);

/* Host-only test hook (no GPU needed): tensor-core engine's input permutation of geometry stage `stage` (0..5) for
 * 1 <= n_kpt <= KPN_MAX_KPT: kmap_out[i] = K index input i is multiplied with, *kbias_out = K index of the bias row,
 * *kpad_out = padded K.  n_inputs must be the stage's input count (stage 0: 7 n_kpt + 64; 1..5: 128, 136, 120, 128, 64). */
int kpn_debug_kmap(int stage, int n_kpt, int n_inputs, int* kmap_out, int* kbias_out, int* kpad_out);

/* Debug hook kept for ABI stability: per-stage cycle stamps of an instrumented build; no instrumented build of the
 * current kernels exists, so it returns KPN_ERR_UNSUPPORTED. */
int kpn_debug_stage_times(kpn_ctx* ctx, unsigned long long* out, int n_words, int* n_tiles);

/* enable != 0: bracket every shading-kernel launch with CUDA events on its stream (no sync). */
int kpn_set_profiling(kpn_ctx* ctx, int enable);

/* Unit test hook for the tensor-core primitive (tests/test_gpu_umma.py): D(128,N) fp32 = A(128,K) fp16 * B(N,K)^T fp16
 * on one warpgroup through wgmma.mma_async (two 64-row MMAs), operands in the shared-memory layouts the kernels use.
 * Device pointers.  N in {16, 32, 48, 64, 96, 112, 128, 144, 192}, K % 16 == 0, K <= 256; variant 0: A from shared memory,
 * variant 1: A from registers, (N, K) = (128, 144) or (64, 128) only. */
int kpn_selftest_umma(int N, int K, const void* A, const void* B, float* D, int variant, void* stream);
/* Same on a 2-CTA cluster: D(256,N) = A(256,K) * B(N,K)^T, each CTA holding half of B's rows and fetching the other half from
 * its peer's shared memory (distributed shared memory) before its wgmma; N in {32, 64, 96, 128, 192}.  The activation tile is
 * d_col 32-bit columns wide with A at columns [a_col, a_col + K/2); mode 0 / 1 / 2: the peer's half is read remotely / pushed
 * by one bulk copy completing on an mbarrier / written by remote stores. */
int kpn_selftest_umma2(int N, int K, const void* A, const void* B, float* D, int a_col, int d_col, int mode, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* KPNERF_B200_H */
