// C ABI of the ray-march path (include/kpnerf_b200.h): context, weight packer, scene packer,
// render / query drivers.  Host logic only; kernels live in kpn_kernels.cu (fp32 SIMT engine)
// and kpn_shade_tc.cu (tensor-core engine).
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <string>
#include <vector>

#include "kpn_launch.h"
#include "kpn_tc.cuh"

using namespace kpn;

namespace {

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = bytes + bytes / 8;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

constexpr int MAX_CHUNKS = 2048;

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

}  // namespace

struct kpn_ctx {
  int device = 0;
  int num_sms = 132;
  std::string err;
  bool have_weights = false, have_scene = false;
  int n_kpt = 0;
  int sp_level = 3;
  float sp_scale = 1.0f, sp_sigma = 0.1f;
  float ani_al = 0.0f;         // mlp_tex.ani_al as set (the kernels see |ani_al|; its gradient needs the sign)

  RawScene* d_raw_scene = nullptr;
  DevScene* d_scene = nullptr;
  RawTarget* d_raw_target = nullptr;
  DevTarget* d_target = nullptr;
  DevWeightsF32* d_wf32 = nullptr;
  DevBuf wbuf;
  DevBuf wblob;                // fp16 weight tiles of the tensor-core engine (core-matrix layout)
  DevBuf wlo;                  // fp16 W_lo tiles of the density-tail stages 4, 5 (same layout as their W_hi tiles)
  TcConsts tcc;                // fp32 constants of the tensor-core engine (kernel parameter)
  bool tc_weights = false;
  int scene_views = 0;
  int map_hw[3][2] = {};       // (H, W) of the bound scene's feat64, feat8, feat_tex
  int* d_counters = nullptr;   // [MAX_CHUNKS] valid samples per shading batch
  int* d_counters2 = nullptr;  // [MAX_CHUNKS] samples that needed a colour (tensor-core engine)
  int counters_used = 0;
  unsigned long long last_total = 0;

  DevBuf stage[4];             // host-sourced maps before packing
  DevBuf atlas[4];             // f64, f8, ftex, img (channel-last fp32)
  DevBuf atlas_fg;
  // per-chunk workspace: rays (origin, dir, near/far), per-ray list ranges of up to two segments, the work list, the compact per-sample
  // records (alpha+sdf, rgb, compositing weight), the fine depths, the colour kernel's latent scratch + work list
  DevBuf ws_rayo, ws_rayd, ws_raynf, ws_rayseg, ws_list, ws_ao, ws_rgb, ws_cw, ws_zfine, ws_lat, ws_list2, ws_ert, ws_contrib, ws_pool;
  DevBuf ws_out, ws_in;
  // kpn_render_rays_backward: staged dL/d outputs, per-list-position gradients (d rad, d sdf | d rgb | a, T), row-major weights,
  // per-CTA gradient slices and their sum, the three feature-map gradients, the front's work list and ray starts before they are
  // put in ray order and the scan scratch that does it
  DevBuf ws_gin, ws_gao, ws_grgb, ws_gat, ws_wr, ws_slices, ws_gred, ws_gmap[3], ws_glist, ws_gscan;
  // marching cubes: per-point vertex offsets, per-cell case bytes and face offsets, scan scratch; the state kpn_mesh_begin
  // leaves for kpn_mesh_emit
  DevBuf mc_vofs, mc_cases, mc_tofs, mc_tmp;
  unsigned long long* d_mc_totals = nullptr;
  unsigned long long* h_mc_totals = nullptr;   // pinned
  const float* mc_field = nullptr;   // the field of the last successful kpn_mesh_begin
  int mc_dims[3] = {0, 0, 0};
  float mc_level = 0.0f;
  long long mc_counts[2] = {0, 0};
  unsigned long long launches = 0;
  bool profiling = false;
  unsigned int* h_wd = nullptr;   // pinned host copy of the tensor-core kernels' watchdog words (refreshed by every render/query)
  std::vector<cudaEvent_t> ev_pool;   // pairs: [2i] start, [2i+1] stop
  size_t ev_used = 0;
};

#define KPN_FAIL(ctx, code, ...)                                   \
  do {                                                             \
    char _b[512];                                                  \
    snprintf(_b, sizeof(_b), __VA_ARGS__);                         \
    (ctx)->err = _b;                                               \
    return (code);                                                 \
  } while (0)

#define KPN_CUDA(ctx, expr)                                                                      \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) KPN_FAIL(ctx, KPN_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

#define KPN_TRY(expr)                  \
  do {                                 \
    int _rc = (expr);                  \
    if (_rc != KPN_OK) return _rc;     \
  } while (0)

static bool mem_ok(int mem) { return mem == KPN_MEM_HOST || mem == KPN_MEM_DEVICE; }

// The host arrays of one call, staged in one device buffer: ws_in for inputs (stage() copies them in), ws_out for outputs
// (unstage() copies them back), so that a call's inputs and outputs never alias.  Every staged array gets the slice at the next
// 256-byte boundary.  stage() reserves the buffer once, for the whole layout, before any copy into it: DevBuf::reserve frees the
// old allocation when it grows.
struct Staging {
  DevBuf* buf;
  bool in, host;   // inputs (ws_in) or outputs (ws_out); the call's arrays are in host memory (KPN_MEM_HOST)
  int n = 0;
  void* ptr[8];
  size_t bytes[8], off[8], total = 0;
  Staging(kpn_ctx* c, bool in, bool host) : buf(in ? &c->ws_in : &c->ws_out), in(in), host(host) {}
  // array p of b bytes: staged when it is a host array, or when `scratch` (the call needs the buffer even if p == nullptr)
  int add(const void* p, size_t b, bool scratch = false) {
    ptr[n] = const_cast<void*>(p);
    bytes[n] = (host && p) || scratch ? b : 0;
    off[n] = total;
    total += (bytes[n] + 255) / 256 * 256;
    return n++;
  }
  // the device pointer the call uses for array i: its slice when staged, else the caller's own pointer
  template <typename T> T* dev(int i) const {
    return static_cast<T*>(bytes[i] ? static_cast<void*>(buf->as<char>() + off[i]) : ptr[i]);
  }
};

static int stage(kpn_ctx* c, const Staging& s, cudaStream_t st) {
  KPN_CUDA(c, s.buf->reserve(s.total));
  for (int i = 0; s.in && i < s.n; ++i)
    if (s.bytes[i] && s.ptr[i]) KPN_CUDA(c, cudaMemcpyAsync(s.dev<void>(i), s.ptr[i], s.bytes[i], cudaMemcpyHostToDevice, st));
  return KPN_OK;
}
static int unstage(kpn_ctx* c, const Staging& s, cudaStream_t st) {
  for (int i = 0; i < s.n; ++i)
    if (s.bytes[i] && s.ptr[i]) KPN_CUDA(c, cudaMemcpyAsync(s.ptr[i], s.dev<void>(i), s.bytes[i], cudaMemcpyDeviceToHost, st));
  return KPN_OK;
}

extern "C" int kpn_abi_version(void) { return KPN_ABI_VERSION; }

extern "C" int kpn_create(int device, kpn_ctx** out) {
  if (!out) return KPN_ERR_ARG;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return KPN_ERR_CUDA;  // no CPU fallback
  if (device < 0 || device >= ndev) return KPN_ERR_ARG;
  kpn_ctx* c = new kpn_ctx();
  c->device = device;
  DeviceGuard g(device);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete c; return KPN_ERR_CUDA; }
  c->num_sms = prop.multiProcessorCount;
  bool ok = cudaMalloc(&c->d_raw_scene, sizeof(RawScene)) == cudaSuccess &&
            cudaMalloc(&c->d_scene, sizeof(DevScene)) == cudaSuccess &&
            cudaMalloc(&c->d_raw_target, sizeof(RawTarget)) == cudaSuccess &&
            cudaMalloc(&c->d_target, sizeof(DevTarget)) == cudaSuccess &&
            cudaMalloc(&c->d_wf32, sizeof(DevWeightsF32)) == cudaSuccess &&
            cudaMalloc(&c->d_counters, sizeof(int) * MAX_CHUNKS) == cudaSuccess &&
            cudaMalloc(&c->d_counters2, sizeof(int) * MAX_CHUNKS) == cudaSuccess &&
            cudaMalloc(&c->d_mc_totals, 2 * sizeof(unsigned long long)) == cudaSuccess &&
            cudaHostAlloc(reinterpret_cast<void**>(&c->h_mc_totals), 2 * sizeof(unsigned long long), cudaHostAllocDefault) == cudaSuccess;
  if (!ok) { kpn_destroy(c); return KPN_ERR_CUDA; }
  cudaMemset(c->d_counters, 0, sizeof(int) * MAX_CHUNKS);
  cudaMemset(c->d_counters2, 0, sizeof(int) * MAX_CHUNKS);
  const size_t wd_bytes = TC_WD_MODULES * TC_WD_WORDS * sizeof(unsigned int);
  if (cudaHostAlloc(reinterpret_cast<void**>(&c->h_wd), wd_bytes, cudaHostAllocDefault) != cudaSuccess) {
    kpn_destroy(c);
    return KPN_ERR_CUDA;
  }
  memset(c->h_wd, 0, wd_bytes);
  *out = c;
  return KPN_OK;
}

extern "C" void kpn_destroy(kpn_ctx* c) {
  if (!c) return;
  DeviceGuard g(c->device);
  cudaFree(c->d_raw_scene); cudaFree(c->d_scene); cudaFree(c->d_raw_target); cudaFree(c->d_target);
  cudaFree(c->d_wf32); cudaFree(c->d_counters); cudaFree(c->d_counters2); cudaFree(c->d_mc_totals);
  if (c->h_mc_totals) cudaFreeHost(c->h_mc_totals);
  c->wbuf.release();
  c->wblob.release();
  c->wlo.release();
  for (auto& b : c->stage) b.release();
  for (auto& b : c->atlas) b.release();
  c->atlas_fg.release();
  for (DevBuf* b : {&c->ws_rayo, &c->ws_rayd, &c->ws_raynf, &c->ws_rayseg, &c->ws_list, &c->ws_ao, &c->ws_rgb, &c->ws_cw, &c->ws_zfine, &c->ws_lat,
                    &c->ws_list2, &c->ws_ert, &c->ws_contrib, &c->ws_pool, &c->ws_out, &c->ws_in, &c->mc_vofs, &c->mc_cases, &c->mc_tofs,
                    &c->mc_tmp, &c->ws_gin, &c->ws_gao, &c->ws_grgb, &c->ws_gat, &c->ws_wr, &c->ws_slices, &c->ws_gred, &c->ws_gmap[0],
                    &c->ws_gmap[1], &c->ws_gmap[2], &c->ws_glist, &c->ws_gscan})
    b->release();
  for (cudaEvent_t e : c->ev_pool) cudaEventDestroy(e);
  if (c->h_wd) cudaFreeHost(c->h_wd);
  delete c;
}

extern "C" const char* kpn_last_error(const kpn_ctx* c) { return c ? c->err.c_str() : "null context"; }

// Stream-ordered copy of every module's watchdog words into out (TC_WD_MODULES x TC_WD_WORDS), and their reset.
static int wd_read(kpn_ctx* c, unsigned int* out, cudaStream_t st) {
  void* w[TC_WD_MODULES];
  KPN_CUDA(c, tc_watchdog_words(w));
  for (int m = 0; m < TC_WD_MODULES; ++m)
    KPN_CUDA(c, cudaMemcpyAsync(out + TC_WD_WORDS * m, w[m], TC_WD_WORDS * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
  return KPN_OK;
}
static int wd_clear(kpn_ctx* c, cudaStream_t st) {
  void* w[TC_WD_MODULES];
  KPN_CUDA(c, tc_watchdog_words(w));
  for (int m = 0; m < TC_WD_MODULES; ++m) KPN_CUDA(c, cudaMemsetAsync(w[m], 0, TC_WD_WORDS * sizeof(unsigned int), st));
  return KPN_OK;
}

// Device watchdog (kpn_tc.cuh): a barrier wait that gives up raises a sticky device flag; every later wait of every later
// tensor-core launch then aborts after a few polls, i.e. the engine keeps producing garbage until the flag is cleared.  Every
// render/query ends with an asynchronous copy of the flag words into pinned host memory (wd_snapshot); every entry point starts
// by looking at the last copy that has landed (wd_check): a raised flag is reported ONCE as KPN_ERR_CUDA and cleared on the
// device (stream-ordered), which re-arms the engine for the calls that follow.
static int wd_check(kpn_ctx* c, cudaStream_t st) {
  volatile unsigned int* w = nullptr;   // the words of the first module whose flag is raised
  for (int m = TC_WD_MODULES - 1; c->h_wd && m >= 0; --m) {
    volatile unsigned int* wm = c->h_wd + TC_WD_WORDS * m;
    if (wm[0] != 0u) w = wm;
  }
  if (!w) return KPN_OK;
  const unsigned int blk = w[1], thr = w[2], tag = w[3], par = w[4];
  for (int i = 0; i < TC_WD_MODULES * TC_WD_WORDS; ++i) c->h_wd[i] = 0u;
  KPN_TRY(wd_clear(c, st));
  KPN_FAIL(c, KPN_ERR_CUDA, "device watchdog: a barrier wait of a tensor-core kernel gave up (block %u, thread %u, tag 0x%x, parity %u); "
           "the results of that call (and of tensor-core calls enqueued after it) are invalid; the flag has been cleared",
           blk, thr, tag, par);
}
static int wd_snapshot(kpn_ctx* c, cudaStream_t st) { return wd_read(c, c->h_wd, st); }

extern "C" int kpn_check_health(kpn_ctx* c, void* stream) {
  if (!c) return KPN_ERR_ARG;
  DeviceGuard g(c->device);
  return wd_check(c, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------
// weights
// ---------------------------------------------------------------------------------------------
static void expected_dims(int n_kpt, int sp_level, int dims[NLAYER][2]) {
  const int enc = (1 + 2 * sp_level) * n_kpt;
  const int t[NLAYER][2] = {{128, enc + 64}, {128, 128}, {120, 136}, {64, 120}, {64, 128}, {64, 64}, {2, 64}, {24, 128},
                            {16, 4}, {35, 16}, {64, 105}, {32, 64}, {32, 32}, {33, 32}, {32, 32}, {1, 32},
                            {16, 37}, {8, 16}, {1, 8}};
  memcpy(dims, t, sizeof(t));
}

// The keypoint-encoding constants of the scene block (sp_scale .. freq), from the weights' sp_args.
static void set_encoding(const kpn_ctx* c, DevScene& h) {
  h.sp_scale = c->sp_scale;
  h.inv2sig2 = 1.0f / (2.0f * c->sp_sigma * c->sp_sigma);
  h.sp_level = c->sp_level;
  double val = 1.0;
  for (int l = 0; l < MAX_SPL; ++l) { h.freq[l] = l < c->sp_level ? (float)(3.14159265358979323846 * val) : 0.0f; val *= 2.0; }
}

extern "C" int kpn_set_weights(kpn_ctx* c, const kpn_weights* w) {
  if (!c || !w) return KPN_ERR_ARG;
  DeviceGuard g(c->device);
  if (w->n_kpt < 1 || w->n_kpt > simt_max_kpt() || w->n_kpt > KPN_MAX_KPT)
    KPN_FAIL(c, KPN_ERR_UNSUPPORTED, "n_kpt=%d unsupported (1..%d)", w->n_kpt, simt_max_kpt());
  if (w->sp_level < 0 || w->sp_level > MAX_SPL || (1 + 2 * w->sp_level) * w->n_kpt + 64 > simt_max_geo_input())
    KPN_FAIL(c, KPN_ERR_UNSUPPORTED, "sp_level=%d unsupported", w->sp_level);
  int dims[NLAYER][2];
  expected_dims(w->n_kpt, w->sp_level, dims);
  size_t total = 0;
  DevWeightsF32 hw;
  std::vector<size_t> woff(NLAYER), boff(NLAYER);
  for (int l = 0; l < NLAYER; ++l) {
    const kpn_layer& L = w->layer[l];
    if (!L.w || !L.bias) KPN_FAIL(c, KPN_ERR_ARG, "layer %d: null weight/bias", l);
    if (L.n_out != dims[l][0] || L.n_in != dims[l][1])
      KPN_FAIL(c, KPN_ERR_ARG, "layer %d: shape (%d,%d) != expected (%d,%d)", l, L.n_out, L.n_in, dims[l][0], dims[l][1]);
    hw.K[l] = L.n_in; hw.N[l] = L.n_out; hw.ldw[l] = (L.n_out + 31) / 32 * 32;
    woff[l] = total; total += (size_t)hw.K[l] * hw.ldw[l];
    boff[l] = total; total += (size_t)hw.ldw[l];
  }
  std::vector<float> host(total, 0.0f);
  std::vector<std::vector<float>> We(NLAYER);  // effective weights, row-major [n_out][n_in]
  for (int l = 0; l < NLAYER; ++l) {
    const kpn_layer& L = w->layer[l];
    We[l].resize((size_t)L.n_out * L.n_in);
    for (int o = 0; o < L.n_out; ++o) {
      double scale = 1.0;
      if (L.g) {  // weight norm, dim=0: w = g * v / ||v||_row  (reference src/utils.py:542-543)
        double nn = 0.0;
        for (int i = 0; i < L.n_in; ++i) nn += (double)L.w[(size_t)o * L.n_in + i] * (double)L.w[(size_t)o * L.n_in + i];
        scale = (double)L.g[o] / std::sqrt(nn);
      }
      for (int i = 0; i < L.n_in; ++i) {
        float e = (float)(scale * (double)L.w[(size_t)o * L.n_in + i]);
        We[l][(size_t)o * L.n_in + i] = e;
        host[woff[l] + (size_t)i * hw.ldw[l] + o] = e;
      }
      host[boff[l] + o] = L.bias[o];
    }
  }
  KPN_CUDA(c, cudaDeviceSynchronize());  // the old buffer may still be in use
  KPN_CUDA(c, c->wbuf.reserve(total * sizeof(float)));
  KPN_CUDA(c, cudaMemcpy(c->wbuf.p, host.data(), total * sizeof(float), cudaMemcpyHostToDevice));
  for (int l = 0; l < NLAYER; ++l) {
    hw.wt[l] = c->wbuf.as<float>() + woff[l];
    hw.bias[l] = c->wbuf.as<float>() + boff[l];
  }
  hw.ani_al_abs = std::fabs(w->ani_al);
  c->ani_al = w->ani_al;
  KPN_CUDA(c, cudaMemcpy(c->d_wf32, &hw, sizeof(hw), cudaMemcpyHostToDevice));
  // ---- tensor-core engine: fp16 weight tiles in the interleaved core-matrix layout + fp32 constants
  c->tc_weights = false;
  if (tc_supported(3, w->n_kpt, w->sp_level)) {
    const TcPlan plan = make_tc_plan(w->n_kpt);
    std::vector<__half> blob(plan.total_bytes / 2, __float2half_rn(0.0f));
    std::vector<__half> lo(tc_weight_lo_bytes(w->n_kpt) / 2, __float2half_rn(0.0f));   // W_lo = fp16(W - W_hi) of stages 4, 5
    // stage -> (layer, first row in the tile); stage 4 stacks the density layer 0 and the colour compress layer
    const int stage_layer[TC_NSTAGE] = {L_GEO0, L_GEO1, L_GEO2, L_GEO3, L_DEN0, L_DEN1, L_BASE0, L_BASE1, L_VIS1A, L_VIS1B, L_VIS2A, L_OUT0, L_RE1};
    auto put_one = [&](int stage, int n, int kk, float wv) {
      const int Np = plan.st[stage].Np;
      const size_t at = (plan.st[stage].off + tc::core_offset_bytes(n, kk, Np)) / 2;
      const __half hi = __float2half_rn(wv);
      blob[at] = hi;
      if (stage == 4 || stage == 5) lo[at - plan.st[4].off / 2] = __float2half_rn(wv - __half2float(hi));
    };
    auto put = [&](int stage, int layer, int row0) {
      const kpn_layer& L = w->layer[layer];
      for (int o = 0; o < L.n_out; ++o) {
        for (int i = 0; i < L.n_in; ++i) {
          put_one(stage, row0 + o, stage < 6 ? tc_kmap(stage, w->n_kpt, i) : i, We[layer][(size_t)o * L.n_in + i]);
        }
        if (stage < 6 || stage == 12) put_one(stage, row0 + o, tc_kbias(stage, w->n_kpt), L.bias[o]);   // bias row (activation column == 1)
      }
    };
    for (int sidx = 0; sidx < TC_NSTAGE; ++sidx) put(sidx, stage_layer[sidx], 0);
    put(4, L_CMP, 64);
    KPN_CUDA(c, c->wblob.reserve(plan.total_bytes));
    KPN_CUDA(c, cudaMemcpy(c->wblob.p, blob.data(), plan.total_bytes, cudaMemcpyHostToDevice));
    KPN_CUDA(c, c->wlo.reserve(lo.size() * 2));
    KPN_CUDA(c, cudaMemcpy(c->wlo.p, lo.data(), lo.size() * 2, cudaMemcpyHostToDevice));
    TcConsts& T = c->tcc;
    memset(&T, 0, sizeof(T));
    auto bias = [&](int layer, float* dst) { for (int o = 0; o < w->layer[layer].n_out; ++o) dst[o] = w->layer[layer].bias[o]; };
    bias(L_BASE0, T.b_base0); bias(L_BASE1, T.b_base1); bias(L_VIS1A, T.b_vis1a); bias(L_VIS1B, T.b_vis1b);
    bias(L_VIS2A, T.b_vis2a); bias(L_OUT0, T.b_out0);
    for (int o = 0; o < 2; ++o) { for (int i = 0; i < 64; ++i) T.w_p2[o][i] = We[L_DEN2][o * 64 + i]; T.b_p2[o] = w->layer[L_DEN2].bias[o]; }
    for (int o = 0; o < 16; ++o) { for (int i = 0; i < 4; ++i) T.w_re0[o][i] = We[L_RE0][o * 4 + i]; T.b_re0[o] = w->layer[L_RE0].bias[o]; }
    for (int i = 0; i < 32; ++i) T.w_vis2b[i] = We[L_VIS2B][i];
    T.b_vis2b = w->layer[L_VIS2B].bias[0];
    for (int o = 0; o < 8; ++o) { for (int i = 0; i < 16; ++i) T.w_out1[o][i] = We[L_OUT1][o * 16 + i]; T.b_out1[o] = w->layer[L_OUT1].bias[o]; }
    for (int i = 0; i < 8; ++i) T.w_out2[i] = We[L_OUT2][i];
    T.b_out2 = w->layer[L_OUT2].bias[0];
    T.ani_abs = std::fabs(w->ani_al);
    c->tc_weights = true;
  }
  const bool same_kpt = c->n_kpt == w->n_kpt;
  c->n_kpt = w->n_kpt; c->sp_level = w->sp_level; c->sp_scale = w->sp_scale; c->sp_sigma = w->sp_sigma;
  c->have_weights = true;
  // A bound scene carries the encoding constants of the weights it was bound with: rewrite them, so that the next render uses
  // the new sp_level / scale / sigma (the device is idle, see above).  Its keypoints can not serve another count: unbind it.
  if (c->have_scene) {
    if (!same_kpt) {
      c->have_scene = false;
    } else {
      DevScene h;
      set_encoding(c, h);
      const size_t lo = offsetof(DevScene, sp_scale), hi = offsetof(DevScene, freq) + sizeof(h.freq);
      KPN_CUDA(c, cudaMemcpy(reinterpret_cast<char*>(c->d_scene) + lo, reinterpret_cast<const char*>(&h) + lo, hi - lo,
                             cudaMemcpyHostToDevice));
    }
  }
  return KPN_OK;
}

// ---------------------------------------------------------------------------------------------
// scene
// ---------------------------------------------------------------------------------------------
static cudaMemcpyKind in_kind(int mem) { return mem == KPN_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice; }

extern "C" int kpn_set_scene(kpn_ctx* c, const kpn_scene* s, void* stream) {
  if (!c || !s) return KPN_ERR_ARG;
  DeviceGuard g(c->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (!c->have_weights) KPN_FAIL(c, KPN_ERR_STATE, "kpn_set_weights must precede kpn_set_scene");
  KPN_TRY(wd_check(c, st));
  if (s->n_views < 1 || s->n_views > KPN_MAX_VIEWS)
    KPN_FAIL(c, KPN_ERR_UNSUPPORTED, "n_views=%d unsupported (1..%d)", s->n_views, KPN_MAX_VIEWS);
  if (s->n_kpt != c->n_kpt) KPN_FAIL(c, KPN_ERR_ARG, "scene n_kpt=%d != weights n_kpt=%d", s->n_kpt, c->n_kpt);
  if (!s->KRT || !s->extrin || !s->kpt3d || !s->bounds || !s->feat64 || !s->feat8 || !s->feat_tex || !s->img)
    KPN_FAIL(c, KPN_ERR_ARG, "null scene pointer");
  if (s->f64_c != 64 || s->f8_c != 8 || s->ftex_c != 8)
    KPN_FAIL(c, KPN_ERR_UNSUPPORTED, "feature channels (%d,%d,%d) != (64,8,8)", s->f64_c, s->f8_c, s->ftex_c);
  if (!mem_ok(s->mem)) KPN_FAIL(c, KPN_ERR_ARG, "bad mem kind");
  const int V = s->n_views;
  cudaMemcpyKind kind = in_kind(s->mem);

  DevScene h;
  memset(&h, 0, sizeof(h));
  h.V = V; h.K = s->n_kpt;
  h.wm1 = s->src_width - 1.0f; h.hm1 = s->src_height - 1.0f;
  h.znear = s->znear; h.zfar = s->zfar;
  h.sdf_invalid = 0.1f / s->nml_scale;
  h.use_fg = s->fg != nullptr;
  set_encoding(c, h);
  struct MapIn { const float* src; int C, H, W, Cp; } maps[4] = {
      {s->feat64, s->f64_c, s->f64_h, s->f64_w, 64}, {s->feat8, s->f8_c, s->f8_h, s->f8_w, 8},
      {s->feat_tex, s->ftex_c, s->ftex_h, s->ftex_w, 8}, {s->img, 3, s->img_h, s->img_w, 4}};
  MapDesc* descs[4] = {&h.f64, &h.f8, &h.ftex, &h.img};
  for (int m = 0; m < 4; ++m) {
    const MapIn& M = maps[m];
    if (M.H < 1 || M.W < 1) KPN_FAIL(c, KPN_ERR_ARG, "map %d has empty extent", m);
    if (m < 3) { c->map_hw[m][0] = M.H; c->map_hw[m][1] = M.W; }
    size_t in_bytes = (size_t)V * M.C * M.H * M.W * sizeof(float);
    size_t out_bytes = (size_t)V * M.Cp * M.H * M.W * sizeof(float);
    if (m < 3 && ((s->layout >> m) & 1)) {
      // already [V][H][W][C] (channels-last encoder output, C == Cp): no re-layout pass.  Device maps are gathered from in
      // place (the caller keeps them alive and unchanged until the next kpn_set_scene); host maps are uploaded as they are.
      const void* ptr = M.src;
      if (s->mem == KPN_MEM_HOST) {
        KPN_CUDA(c, c->atlas[m].reserve(out_bytes));
        KPN_CUDA(c, cudaMemcpyAsync(c->atlas[m].p, M.src, in_bytes, cudaMemcpyHostToDevice, st));
        ptr = c->atlas[m].p;
      }
      descs[m]->ptr = ptr; descs[m]->C = M.Cp; descs[m]->H = M.H; descs[m]->W = M.W;
      continue;
    }
    const float* dsrc = M.src;
    if (s->mem == KPN_MEM_HOST) {
      KPN_CUDA(c, c->stage[m].reserve(in_bytes));
      KPN_CUDA(c, cudaMemcpyAsync(c->stage[m].p, M.src, in_bytes, cudaMemcpyHostToDevice, st));
      dsrc = c->stage[m].as<float>();
    }
    KPN_CUDA(c, c->atlas[m].reserve(out_bytes));
    KPN_CUDA(c, launch_pack_nhwc_f32(dsrc, c->atlas[m].as<float>(), V, M.C, M.H, M.W, M.Cp, st));
    c->launches++;
    descs[m]->ptr = c->atlas[m].p; descs[m]->C = M.Cp; descs[m]->H = M.H; descs[m]->W = M.W;
  }
  if (s->fg) {
    size_t bytes = (size_t)V * s->fg_h * s->fg_w;
    KPN_CUDA(c, c->atlas_fg.reserve(bytes));
    KPN_CUDA(c, cudaMemcpyAsync(c->atlas_fg.p, s->fg, bytes, kind, st));
    h.fg.ptr = c->atlas_fg.p; h.fg.C = 1; h.fg.H = s->fg_h; h.fg.W = s->fg_w;
  }
  KPN_CUDA(c, cudaMemcpyAsync(c->d_scene, &h, sizeof(h), cudaMemcpyHostToDevice, st));
  KPN_CUDA(c, cudaMemcpyAsync(c->d_raw_scene->KRT, s->KRT, sizeof(float) * 16 * V, kind, st));
  KPN_CUDA(c, cudaMemcpyAsync(c->d_raw_scene->extrin, s->extrin, sizeof(float) * 16 * V, kind, st));
  KPN_CUDA(c, cudaMemcpyAsync(c->d_raw_scene->kpt3d, s->kpt3d, sizeof(float) * 3 * s->n_kpt, kind, st));
  KPN_CUDA(c, cudaMemcpyAsync(c->d_raw_scene->bounds, s->bounds, sizeof(float) * 6, kind, st));
  KPN_CUDA(c, launch_prep_scene(c->d_raw_scene, c->d_scene, st));
  c->launches++;
  if (s->fg) { KPN_CUDA(c, launch_fg_box(c->d_scene, V, st)); c->launches++; }
  c->have_scene = true;
  c->scene_views = V;
  return KPN_OK;
}

// ---------------------------------------------------------------------------------------------
// shading of a batch of samples with the selected engine
// ---------------------------------------------------------------------------------------------
// Shades the samples of list[0 .. *counter) (device-side count, at most n) with the selected engine; `so` says where the results go.
static int shade_batch(kpn_ctx* c, const SampleSrc& src, const int* list, const int* counter, int* counter2, long long n,
                       int query_mode, const ShadeOut& so, int engine, cudaStream_t st) {
  const bool use_tc = engine != 1;
  if (engine < 0 || engine > 4) KPN_FAIL(c, KPN_ERR_ARG, "kpn_opts.engine = %d (0 .. 4)", engine);
  if (use_tc && !(c->tc_weights && tc_supported(c->scene_views, c->n_kpt, c->sp_level)))
    KPN_FAIL(c, KPN_ERR_UNSUPPORTED, "the tensor-core engine covers n_views 3 or 4, 1 <= n_kpt <= %d, sp_level == 3; this scene has "
             "n_views=%d n_kpt=%d sp_level=%d: request engine = 1 (fp32 CUDA-core engine, ~25x slower) explicitly",
             KPN_MAX_KPT, c->scene_views, c->n_kpt, c->sp_level);
  cudaEvent_t e0 = nullptr, em = nullptr, e1 = nullptr;   // start | after the geometry kernel | stop
  if (c->profiling) {
    while (c->ev_used + 3 > c->ev_pool.size()) {
      cudaEvent_t a;
      KPN_CUDA(c, cudaEventCreate(&a));
      c->ev_pool.push_back(a);
    }
    e0 = c->ev_pool[c->ev_used]; em = c->ev_pool[c->ev_used + 1]; e1 = c->ev_pool[c->ev_used + 2];
    c->ev_used += 3;
    KPN_CUDA(c, cudaEventRecord(e0, st));
  }
  if (use_tc) {
    KPN_CUDA(c, c->ws_lat.reserve((size_t)n * 48));
    KPN_CUDA(c, c->ws_list2.reserve((size_t)n * 8));
    KPN_CUDA(c, c->ws_pool.reserve(tc_pool_bytes(n)));
  }
  ShadeBatch b;
  b.sc = c->d_scene; b.n_views = c->scene_views; b.n_kpt = c->n_kpt;
  b.src = src; b.list = list; b.counter = counter; b.n_max = n; b.query_mode = query_mode; b.so = so;
  b.num_sms = c->num_sms; b.st = st;
  b.wf32 = c->d_wf32;
  b.tcc = &c->tcc; b.wblob = c->wblob.as<uint8_t>(); b.wlo = c->wlo.as<uint8_t>();
  b.lo_mask = engine == 2 ? 0xC0 : 0xF0;   // single-term weights (engine 2) keep the A_lo passes only
  b.lat = c->ws_lat.as<uint4>(); b.pool = c->ws_pool.as<float>(); b.list2 = c->ws_list2.as<int2>(); b.count2 = counter2;
  b.after_geo = em; b.launches = &c->launches;
  KPN_CUDA(c, use_tc ? launch_shade_tc(b) : launch_shade_simt(b));
  if (c->profiling) KPN_CUDA(c, cudaEventRecord(e1, st));
  return KPN_OK;
}

// rays per chunk: bounded by the per-sample workspace; fewer, larger launches amortise the persistent kernels' prologue (weight
// load) and tail (measured 4 / 8 / 32 Mi samples: 30.5 / 30.2 / 30.0 ms per 512x512x128 frame).  KPN_CHUNK_SAMPLES overrides
// the default of 32 Mi samples.
static long long chunk_rays(long long R, int Smax) {
  static const long long chunk_samples = [] {
    const char* e = getenv("KPN_CHUNK_SAMPLES");
    long long v = e ? atoll(e) : 0;
    return v >= (1ll << 16) && v <= (1ll << 28) ? v : (32ll << 20);
  }();
  long long Rc = chunk_samples / Smax;
  Rc = (Rc / 128) * 128;
  if (Rc < 128) Rc = 128;
  return Rc > R ? R : Rc;
}

// every per-chunk workspace buffer of a render of Rc rays x (Sc coarse, Smax total) samples
static int reserve_render(kpn_ctx* c, long long Rc, int Sc, int Smax, bool fine, bool contrib, bool ert) {
  const size_t n = (size_t)Rc * Smax;
  KPN_CUDA(c, c->ws_rayo.reserve((size_t)Rc * 3 * sizeof(float)));
  KPN_CUDA(c, c->ws_rayd.reserve((size_t)Rc * 3 * sizeof(float)));
  KPN_CUDA(c, c->ws_raynf.reserve((size_t)Rc * 4 * sizeof(float)));   // clipped near/far | a lattice's near/far before the clip
  KPN_CUDA(c, c->ws_rayseg.reserve((size_t)Rc * 4 * sizeof(int)));   // start | cnt of segment 0, start | cnt of segment 1
  KPN_CUDA(c, c->ws_list.reserve(n * sizeof(int)));
  KPN_CUDA(c, c->ws_ao.reserve(n * sizeof(float2)));
  KPN_CUDA(c, c->ws_rgb.reserve(n * 3 * sizeof(float)));
  KPN_CUDA(c, c->ws_lat.reserve(n * 48));
  KPN_CUDA(c, c->ws_list2.reserve(n * 8));
  if (fine || contrib) KPN_CUDA(c, c->ws_cw.reserve((size_t)Rc * Sc * sizeof(float)));
  if (contrib) KPN_CUDA(c, c->ws_contrib.reserve((size_t)Rc * Sc * sizeof(float)));
  if (fine) KPN_CUDA(c, c->ws_zfine.reserve(n * sizeof(float)));
  if (ert) KPN_CUDA(c, c->ws_ert.reserve((size_t)Rc * sizeof(float)));
  return KPN_OK;
}

constexpr int OUT_W[7] = {3, 1, 1, 3, 1, 1, 1};   // floats per ray of the kpn_out planes tex_fg .. sdf
constexpr int RAY_W[3] = {3, 3, 2};               // floats per ray of origins, dirs, near/far

// The staging of n per-ray float arrays of R rays, a[i] with w[i] floats per ray: a render's kpn_out planes, kpn_render_rays'
// inputs, kpn_camera_rays' outputs.  a == nullptr: room for every array, the most a render stages.
static Staging ray_planes(kpn_ctx* c, bool in, bool host, long long R, int n, const int* w, const float* const* a) {
  Staging s(c, in, host);
  for (int i = 0; i < n; ++i) s.add(a ? a[i] : nullptr, (size_t)w[i] * R * sizeof(float), !a);
  return s;
}

extern "C" int kpn_reserve(kpn_ctx* c, long long max_rays, int max_samples) {
  if (!c || max_rays < 1 || max_samples < 1) return KPN_ERR_ARG;
  DeviceGuard g(c->device);
  const long long Rc = chunk_rays(max_rays, max_samples);
  KPN_TRY(reserve_render(c, Rc, max_samples, max_samples, true, true, true));
  // the host staging of the outputs and of kpn_render_rays' inputs, laid out as a render lays them out
  KPN_CUDA(c, c->ws_out.reserve(ray_planes(c, false, true, max_rays, 7, OUT_W, nullptr).total));
  KPN_CUDA(c, c->ws_in.reserve(ray_planes(c, true, true, max_rays, 3, RAY_W, nullptr).total));
  return KPN_OK;
}

static int begin_counters(kpn_ctx* c, cudaStream_t st) {
  KPN_CUDA(c, cudaMemsetAsync(c->d_counters, 0, sizeof(int) * MAX_CHUNKS, st));
  KPN_CUDA(c, cudaMemsetAsync(c->d_counters2, 0, sizeof(int) * MAX_CHUNKS, st));
  c->counters_used = 0;
  c->last_total = 0;
  return KPN_OK;
}

// Target camera -> device constants (d_target); with_scene: also the bound scene's foreground windows.
static int upload_target(kpn_ctx* c, const kpn_target* tg, bool with_scene, cudaStream_t st) {
  cudaMemcpyKind kind = in_kind(tg->mem);
  KPN_CUDA(c, cudaMemcpyAsync(c->d_raw_target->K, tg->K, sizeof(float) * 16, kind, st));
  KPN_CUDA(c, cudaMemcpyAsync(c->d_raw_target->RT, tg->RT, sizeof(float) * 16, kind, st));
  DevTarget ht;
  memset(&ht, 0, sizeof(ht));
  ht.znear = tg->znear; ht.zfar = tg->zfar; ht.x0 = tg->x0; ht.y0 = tg->y0; ht.step = tg->step; ht.nx = tg->nx; ht.ny = tg->ny;
  ht.step_y = tg->step_y > 0 ? tg->step_y : tg->step;
  KPN_CUDA(c, cudaMemcpyAsync(c->d_target, &ht, sizeof(ht), cudaMemcpyHostToDevice, st));
  KPN_CUDA(c, launch_prep_target(c->d_raw_target, c->d_target, with_scene ? c->d_scene : nullptr, st));
  c->launches++;
  return KPN_OK;
}

// The rays a render marches: the pixel lattice of the target in d_target (lattice), or explicit device arrays o, d (R,3) and
// nf (R,2, near/far before the bounding-box clip).
struct RaySource {
  bool lattice;
  const float* o;
  const float* d;
  const float* nf;
};

// The render of R rays x (S_c [+ S_f]) samples shared by kpn_render and kpn_render_rays: chunks of rays, each through the coarse
// pass, the resampling and the fine pass; outputs are planes of R values (kpn_out).  Arguments are checked by the caller.
static int render_rays(kpn_ctx* c, long long R, const RaySource& rays, const kpn_opts* op, const kpn_out* out, cudaStream_t st) {
  const int Sc = op->sample_per_ray_c, Sf = op->fine ? op->sample_per_ray_f : 0;
  const int Smax = Sc + Sf;
  // outputs: render into device planes, copy to the host at the end if requested
  const float* user[7] = {out->tex_fg, out->depth, out->alpha, out->tex_fg_fine, out->depth_fine, out->alpha_fine, out->sdf};
  const bool host_out = out->mem == KPN_MEM_HOST;
  const Staging outs = ray_planes(c, false, host_out, R, 7, OUT_W, user);
  KPN_TRY(stage(c, outs, st));
  float* dev[7];
  for (int i = 0; i < 7; ++i) dev[i] = outs.dev<float>(i);

  const long long Rc = chunk_rays(R, Smax);
  const long long nchunks = (R + Rc - 1) / Rc;
  if (nchunks * 4 > MAX_CHUNKS) KPN_FAIL(c, KPN_ERR_ARG, "frame too large for one call (%lld chunks)", nchunks);
  const bool need_contrib = op->fine || out->contrib;
  const bool ert_on = op->ert_eps > 0.0f;
  KPN_TRY(reserve_render(c, Rc, Sc, Smax, op->fine != 0, need_contrib, ert_on));
  KPN_TRY(begin_counters(c, st));
  cudaMemcpyKind okind = host_out ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  int* seg = c->ws_rayseg.as<int>();
  int* list = c->ws_list.as<int>();
  float2* ao = c->ws_ao.as<float2>();
  float* rgbw = c->ws_rgb.as<float>();
  const float* ro = nullptr;   // the current chunk's rays
  const float* rd = nullptr;
  const float* rnf = nullptr;
  // One pass over nr rays x S samples (zbuf == nullptr: the coarse pass, uniform depths): front (rays + validity + ray-ordered
  // work list) -> shading -> compositing.  Early-ray termination (ert_eps > 0, S >= 8): the front half of every ray is shaded
  // and composited first; rays whose transmittance behind it is < ert_eps get no entries for the back half (their remaining
  // contribution to any channel is < ert_eps; the reference has no such option, ert_eps = 0 reproduces it exactly).  The
  // back half's entries live in the list range [nr*half, nr*S) and have their own per-ray ranges (segment 1).
  auto pass = [&](int r0, int nr, int S, const float* zbuf, int slot, float* color, float* depth, float* alpha, float* sdf,
                  float* cw) -> int {
    SampleSrc src;
    memset(&src, 0, sizeof(src));
    src.mode = 0; src.S = S; src.ray_d = rd; src.z = zbuf; src.ray_nf = c->ws_raynf.as<float>(); src.o = ro;
    const long long n = (long long)nr * S;
    int* start0 = seg; int* cnt0 = seg + Rc; int* start1 = seg + 2 * Rc; int* cnt1 = seg + 3 * Rc;
    const bool two = ert_on && S >= 8;
    const int half = S / 2;
    ShadeOut so;
    memset(&so, 0, sizeof(so));
    so.ao = ao; so.rgb = rgbw;
    KPN_CUDA(c, launch_front(c->d_scene, c->d_target, nr, S, zbuf, ro, rd, rnf, c->ws_raynf.as<float>(), list, 0, c->d_counters + slot,
                             start0, cnt0, two ? ErtSegment{0, half, nullptr, 0.0f} : ErtSegment{0, 0, nullptr, 0.0f}, st));
    c->launches++;
    so.list_base = 0;
    KPN_TRY(shade_batch(c, src, list, c->d_counters + slot, c->d_counters2 + slot, two ? (long long)nr * half : n, 0, so, op->engine, st));
    if (two) {
      KPN_CUDA(c, launch_composite(list, ao, rgbw, start0, cnt0, nullptr, nullptr, zbuf, c->ws_raynf.as<float>(), r0, nr, S, R, nullptr,
                                   nullptr, nullptr, nullptr, c->ws_ert.as<float>(), nullptr, st));
      const int base1 = nr * half;
      KPN_CUDA(c, launch_front(c->d_scene, c->d_target, nr, S, zbuf, ro, rd, rnf, c->ws_raynf.as<float>(), list, base1,
                               c->d_counters + slot + 1, start1, cnt1, ErtSegment{half, S, c->ws_ert.as<float>(), op->ert_eps}, st));
      c->launches += 2;
      so.list_base = base1;
      KPN_TRY(shade_batch(c, src, list + base1, c->d_counters + slot + 1, c->d_counters2 + slot + 1, n - base1, 0, so, op->engine, st));
    }
    KPN_CUDA(c, launch_composite(list, ao, rgbw, start0, cnt0, two ? start1 : nullptr, two ? cnt1 : nullptr, zbuf, c->ws_raynf.as<float>(),
                                 r0, nr, S, R, color, depth, alpha, sdf, nullptr, cw, st));
    c->launches++;
    return KPN_OK;
  };

  for (long long ch = 0; ch < nchunks; ++ch) {
    const long long r0 = ch * Rc;
    const int nr = (int)((R - r0) < Rc ? (R - r0) : Rc);
    if (rays.lattice) {
      ro = c->ws_rayo.as<float>(); rd = c->ws_rayd.as<float>(); rnf = c->ws_raynf.as<float>() + 2 * Rc;
      KPN_CUDA(c, launch_camera_rays(c->d_target, r0, nr, c->ws_rayo.as<float>(), c->ws_rayd.as<float>(), c->ws_raynf.as<float>() + 2 * Rc, st));
      c->launches++;
    } else {
      ro = rays.o + 3 * r0; rd = rays.d + 3 * r0; rnf = rays.nf + 2 * r0;
    }
    // coarse pass; with early-ray termination its weights must still cover every sample of the ray for the resampling pass:
    // rays that terminated early simply have zero weight behind the cut
    KPN_TRY(pass((int)r0, nr, Sc, nullptr, (int)(4 * ch), dev[0], dev[1], dev[2], nullptr, need_contrib ? c->ws_cw.as<float>() : nullptr));
    c->last_total += (unsigned long long)nr * Sc;
    if (need_contrib) {
      // dense weights (debug output) and / or the resampled + merged depths of the fine pass, one warp per ray
      const bool two = ert_on && Sc >= 8;
      float* zout = (op->fine && !op->z_fine_override) ? c->ws_zfine.as<float>() : nullptr;
      float* cden = out->contrib ? c->ws_contrib.as<float>() : nullptr;
      if (zout || cden) {
        KPN_CUDA(c, launch_resample(list, c->ws_cw.as<float>(), seg, seg + Rc, two ? seg + 2 * Rc : nullptr, two ? seg + 3 * Rc : nullptr,
                                    c->ws_raynf.as<float>(), nr, Sc, zout ? Sf : 0, zout, cden, st));
        c->launches++;
      }
      if (out->contrib)
        KPN_CUDA(c, cudaMemcpyAsync(out->contrib + r0 * Sc, c->ws_contrib.p, (size_t)nr * Sc * sizeof(float), okind, st));
    }
    if (op->fine) {
      if (op->z_fine_override)
        KPN_CUDA(c, cudaMemcpyAsync(c->ws_zfine.p, op->z_fine_override + r0 * Smax, (size_t)nr * Smax * sizeof(float),
                                    in_kind(out->mem), st));
      KPN_TRY(pass((int)r0, nr, Smax, c->ws_zfine.as<float>(), (int)(4 * ch + 2), dev[3], dev[4], dev[5], dev[6], nullptr));
      c->last_total += (unsigned long long)nr * Smax;
      if (out->z_fine)
        KPN_CUDA(c, cudaMemcpyAsync(out->z_fine + r0 * Smax, c->ws_zfine.p, (size_t)nr * Smax * sizeof(float), okind, st));
    }
  }
  c->counters_used = (int)(4 * nchunks);
  KPN_TRY(unstage(c, outs, st));
  return wd_snapshot(c, st);
}


static int check_target(kpn_ctx* c, const kpn_target* tg) {
  if (tg->nx < 1 || tg->ny < 1 || tg->step < 1 || tg->step_y < 0) KPN_FAIL(c, KPN_ERR_ARG, "empty pixel lattice");
  if (!tg->K || !tg->RT) KPN_FAIL(c, KPN_ERR_ARG, "null target camera");
  return KPN_OK;
}

// The options and limits of a render of R rays, shared by kpn_render (tg: its target, whose lattice is checked here too) and
// kpn_render_rays (tg == nullptr): the sample counts, at most 2^31 - 1 rays (the compositing kernel indexes the output planes
// with an int) and 2^40 samples, and the memory kinds of the target and the outputs.
static int check_render(kpn_ctx* c, const kpn_opts* op, const kpn_target* tg, long long R, const kpn_out* out) {
  const int Sc = op->sample_per_ray_c, Sf = op->fine ? op->sample_per_ray_f : 0;
  if (Sc < 1 || Sc > max_coarse_samples()) KPN_FAIL(c, KPN_ERR_ARG, "sample_per_ray_c=%d out of range", Sc);
  if (op->fine && (Sc < 3 || Sf < 1 || Sf > 1024)) KPN_FAIL(c, KPN_ERR_ARG, "fine pass needs S_c>=3 and 1<=S_f<=1024");
  if (tg) KPN_TRY(check_target(c, tg));
  if (R > 0x7fffffffll || R * (Sc + Sf) >= (1ll << 40)) KPN_FAIL(c, KPN_ERR_ARG, "too many rays / samples (%lld rays)", R);
  if (!mem_ok(out->mem) || (tg && !mem_ok(tg->mem))) KPN_FAIL(c, KPN_ERR_ARG, "bad mem kind");
  return KPN_OK;
}

extern "C" int kpn_render(kpn_ctx* c, const kpn_target* tg, const kpn_opts* op, const kpn_out* out, void* stream) {
  if (!c || !tg || !op || !out) return KPN_ERR_ARG;
  DeviceGuard g(c->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (!c->have_scene) KPN_FAIL(c, KPN_ERR_STATE, "kpn_set_scene must precede kpn_render");
  KPN_TRY(wd_check(c, st));
  const long long R = (long long)tg->nx * tg->ny;
  KPN_TRY(check_render(c, op, tg, R, out));
  KPN_TRY(upload_target(c, tg, true, st));
  return render_rays(c, R, RaySource{true, nullptr, nullptr, nullptr}, op, out, st);
}

extern "C" int kpn_render_rays(kpn_ctx* c, const kpn_rays* rays, const kpn_opts* op, const kpn_out* out, void* stream) {
  if (!c || !rays || !op || !out || rays->n < 0) return KPN_ERR_ARG;
  if (rays->n == 0) return KPN_OK;
  DeviceGuard g(c->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (!rays->origins || !rays->dirs || !rays->near_far) KPN_FAIL(c, KPN_ERR_ARG, "null ray arrays");
  if (!mem_ok(rays->mem)) KPN_FAIL(c, KPN_ERR_ARG, "bad mem kind");
  if (!c->have_scene) KPN_FAIL(c, KPN_ERR_STATE, "kpn_set_scene must precede kpn_render_rays");
  KPN_TRY(wd_check(c, st));
  const long long R = rays->n;
  KPN_TRY(check_render(c, op, nullptr, R, out));
  const float* a[3] = {rays->origins, rays->dirs, rays->near_far};
  const Staging in = ray_planes(c, true, rays->mem == KPN_MEM_HOST, R, 3, RAY_W, a);
  KPN_TRY(stage(c, in, st));
  KPN_CUDA(c, launch_prep_target(nullptr, c->d_target, c->d_scene, st));   // the scene's foreground windows only
  c->launches++;
  return render_rays(c, R, RaySource{false, in.dev<const float>(0), in.dev<const float>(1), in.dev<const float>(2)}, op, out, st);
}

// The packed gradient vector of the bound weights: every layer's dW (n_out, n_in), its db, then d ani_al.
static GradLayout grad_layout(const kpn_ctx* c) {
  int dims[NLAYER][2];
  expected_dims(c->n_kpt, c->sp_level, dims);
  GradLayout g;
  int off = 0;
  for (int l = 0; l < NLAYER; ++l) { g.wo[l] = off; off += dims[l][0] * dims[l][1]; }
  for (int l = 0; l < NLAYER; ++l) { g.bo[l] = off; off += dims[l][0]; }
  g.ani = off;
  g.total = off + 1;
  return g;
}

extern "C" int kpn_render_rays_backward(kpn_ctx* c, const kpn_rays* rays, const kpn_opts* op, const kpn_out* gout, const kpn_grads* gr,
                                        void* stream) {
  if (!c || !rays || !op || !gout || !gr || rays->n < 0) return KPN_ERR_ARG;
  DeviceGuard g(c->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (rays->n > 0 && (!rays->origins || !rays->dirs || !rays->near_far)) KPN_FAIL(c, KPN_ERR_ARG, "null ray arrays");
  if (!mem_ok(rays->mem) || !mem_ok(gout->mem) || !mem_ok(gr->mem)) KPN_FAIL(c, KPN_ERR_ARG, "bad mem kind");
  for (int l = 0; l < NLAYER; ++l)
    if (!gr->dW[l] || !gr->db[l]) KPN_FAIL(c, KPN_ERR_ARG, "null gradient of layer %d", l);
  if (!gr->d_ani_al || !gr->d_feat64 || !gr->d_feat8 || !gr->d_feat_tex) KPN_FAIL(c, KPN_ERR_ARG, "null gradient array");
  if (!c->have_weights || !c->have_scene) KPN_FAIL(c, KPN_ERR_STATE, "kpn_set_weights and kpn_set_scene must precede kpn_render_rays_backward");
  if (op->ert_eps > 0.0f)
    KPN_FAIL(c, KPN_ERR_UNSUPPORTED, "ert_eps > 0: the samples early-ray termination skips have gradients; differentiate with ert_eps = 0");
  KPN_TRY(wd_check(c, st));
  const long long R = rays->n;
  KPN_TRY(check_render(c, op, nullptr, R, gout));
  const int Sc = op->sample_per_ray_c, Sf = op->fine ? op->sample_per_ray_f : 0;
  const int Smax = Sc + Sf;
  const float* a[3] = {rays->origins, rays->dirs, rays->near_far};
  const Staging in = ray_planes(c, true, rays->mem == KPN_MEM_HOST, R, 3, RAY_W, a);
  KPN_TRY(stage(c, in, st));
  const float* gplane[7] = {gout->tex_fg, gout->depth, gout->alpha, gout->tex_fg_fine, gout->depth_fine, gout->alpha_fine, gout->sdf};
  Staging gin = ray_planes(c, true, gout->mem == KPN_MEM_HOST, R, 7, OUT_W, gplane);
  gin.buf = &c->ws_gin;
  KPN_TRY(stage(c, gin, st));
  const float* gdev[7];
  for (int i = 0; i < 7; ++i) gdev[i] = gin.dev<const float>(i);

  // gradient accumulators: one slice per CTA of the shading backward, the feature maps, the row-major weights
  const GradLayout lay = grad_layout(c);
  const int V = c->scene_views;
  const int map_c[3] = {64, 8, 8};
  KPN_CUDA(c, c->ws_wr.reserve((size_t)lay.total * sizeof(float)));
  KPN_CUDA(c, c->ws_slices.reserve((size_t)c->num_sms * lay.total * sizeof(float)));
  KPN_CUDA(c, c->ws_gred.reserve((size_t)lay.total * sizeof(float)));
  KPN_CUDA(c, cudaMemsetAsync(c->ws_slices.p, 0, (size_t)c->num_sms * lay.total * sizeof(float), st));
  size_t map_bytes[3];
  for (int m = 0; m < 3; ++m) {
    map_bytes[m] = (size_t)V * c->map_hw[m][0] * c->map_hw[m][1] * map_c[m] * sizeof(float);
    KPN_CUDA(c, c->ws_gmap[m].reserve(map_bytes[m]));
    KPN_CUDA(c, cudaMemsetAsync(c->ws_gmap[m].p, 0, map_bytes[m], st));
  }
  KPN_CUDA(c, launch_weights_rowmajor(c->d_wf32, c->ws_wr.as<float>(), lay, st));
  c->launches++;
  KPN_CUDA(c, launch_prep_target(nullptr, c->d_target, c->d_scene, st));   // the scene's foreground windows only
  c->launches++;

  const long long Rc = chunk_rays(R > 0 ? R : 1, Smax);
  const long long nchunks = (R + Rc - 1) / Rc;
  if (nchunks * 4 > MAX_CHUNKS) KPN_FAIL(c, KPN_ERR_ARG, "batch too large for one call (%lld chunks)", nchunks);
  KPN_TRY(reserve_render(c, Rc, Sc, Smax, op->fine != 0, op->fine != 0, false));
  const size_t n = (size_t)Rc * Smax;
  KPN_CUDA(c, c->ws_gao.reserve(n * sizeof(float2)));
  KPN_CUDA(c, c->ws_grgb.reserve(n * 3 * sizeof(float)));
  KPN_CUDA(c, c->ws_gat.reserve(n * sizeof(float2)));
  KPN_CUDA(c, c->ws_glist.reserve((n + (size_t)Rc) * sizeof(int)));
  const size_t scan_bytes = canonical_list_temp_bytes((int)Rc);
  KPN_CUDA(c, c->ws_gscan.reserve(scan_bytes));
  KPN_TRY(begin_counters(c, st));
  int* seg = c->ws_rayseg.as<int>();
  int* list = c->ws_list.as<int>();
  float2* ao = c->ws_ao.as<float2>();
  float* rgbw = c->ws_rgb.as<float>();
  float* raynf = c->ws_raynf.as<float>();
  ShadeGrad sg;
  sg.d_ao = c->ws_gao.as<float2>(); sg.d_rgb = c->ws_grgb.as<float>(); sg.wr = c->ws_wr.as<float>(); sg.lay = lay;
  sg.slices = c->ws_slices.as<float>();
  sg.d_f64 = c->ws_gmap[0].as<float>(); sg.d_f8 = c->ws_gmap[1].as<float>(); sg.d_ftex = c->ws_gmap[2].as<float>();
  sg.ani_sign = c->ani_al > 0.0f ? 1.0f : (c->ani_al < 0.0f ? -1.0f : 0.0f);
  // One pass over nr rays x S samples with the fp32 engine (the recorded forward), then its backward: compositing, shading.  The
  // front's work list is put in ray order first (launch_canonical_list): which samples share a tile of the shading backward, and
  // so the summation order of dW, db and d ani_al, then depends on the rays alone and not on the order in which the front's
  // blocks won their atomics.
  int* raw_list = c->ws_glist.as<int>();
  int* raw_start = raw_list + n;
  auto pass = [&](const float* ro, const float* rd, const float* rnf, int r0, int nr, int S, const float* zbuf, int slot, const RayGrad& rg,
                  float* cw) -> int {
    SampleSrc src;
    memset(&src, 0, sizeof(src));
    src.mode = 0; src.S = S; src.ray_d = rd; src.z = zbuf; src.ray_nf = raynf; src.o = ro;
    ShadeOut so;
    memset(&so, 0, sizeof(so));
    so.ao = ao; so.rgb = rgbw;
    KPN_CUDA(c, launch_front(c->d_scene, c->d_target, nr, S, zbuf, ro, rd, rnf, raynf, raw_list, 0, c->d_counters + slot, raw_start,
                             seg + Rc, ErtSegment{0, 0, nullptr, 0.0f}, st));
    KPN_CUDA(c, launch_canonical_list(raw_list, raw_start, seg + Rc, nr, list, seg, c->ws_gscan.p, scan_bytes, c->num_sms, st));
    c->launches += 3;
    KPN_TRY(shade_batch(c, src, list, c->d_counters + slot, c->d_counters2 + slot, (long long)nr * S, 0, so, 1, st));
    if (cw) {
      KPN_CUDA(c, launch_composite(list, ao, rgbw, seg, seg + Rc, nullptr, nullptr, zbuf, raynf, r0, nr, S, R, nullptr, nullptr, nullptr,
                                   nullptr, nullptr, cw, st));
      c->launches++;
    }
    KPN_CUDA(c, launch_composite_backward(list, ao, rgbw, seg, seg + Rc, zbuf, raynf, r0, nr, S, R, rg, c->ws_gao.as<float2>(),
                                          c->ws_grgb.as<float>(), c->ws_gat.as<float2>(), c->num_sms, st));
    ShadeBatch b;
    memset(&b, 0, sizeof(b));
    b.sc = c->d_scene; b.n_views = V; b.n_kpt = c->n_kpt; b.src = src; b.list = list; b.counter = c->d_counters + slot;
    b.n_max = (long long)nr * S; b.so = so; b.num_sms = c->num_sms; b.st = st; b.wf32 = c->d_wf32; b.launches = &c->launches;
    KPN_CUDA(c, launch_shade_simt_backward(b, sg));
    c->launches++;
    return KPN_OK;
  };
  for (long long ch = 0; ch < nchunks; ++ch) {
    const long long r0 = ch * Rc;
    const int nr = (int)((R - r0) < Rc ? (R - r0) : Rc);
    const float* ro = in.dev<const float>(0) + 3 * r0;
    const float* rd = in.dev<const float>(1) + 3 * r0;
    const float* rnf = in.dev<const float>(2) + 2 * r0;
    // coarse pass: its compositing weights drive the resampling (the fine depths carry no gradient, as under the reference's
    // torch.no_grad), so the fine depths are computed before its list is overwritten
    KPN_TRY(pass(ro, rd, rnf, (int)r0, nr, Sc, nullptr, (int)(4 * ch), RayGrad{gdev[0], gdev[2], gdev[1], nullptr},
                 op->fine ? c->ws_cw.as<float>() : nullptr));
    c->last_total += (unsigned long long)nr * Sc;
    if (op->fine) {
      if (op->z_fine_override) {
        KPN_CUDA(c, cudaMemcpyAsync(c->ws_zfine.p, op->z_fine_override + r0 * Smax, (size_t)nr * Smax * sizeof(float),
                                    in_kind(gout->mem), st));
      } else {
        KPN_CUDA(c, launch_resample(list, c->ws_cw.as<float>(), seg, seg + Rc, nullptr, nullptr, raynf, nr, Sc, Sf, c->ws_zfine.as<float>(),
                                    nullptr, st));
        c->launches++;
      }
      KPN_TRY(pass(ro, rd, rnf, (int)r0, nr, Smax, c->ws_zfine.as<float>(), (int)(4 * ch + 2),
                   RayGrad{gdev[3], gdev[5], gdev[4], gdev[6]}, nullptr));
      c->last_total += (unsigned long long)nr * Smax;
    }
  }
  c->counters_used = (int)(4 * nchunks);
  KPN_CUDA(c, launch_grad_reduce(c->ws_slices.as<float>(), c->num_sms, lay.total, c->ws_gred.as<float>(), st));
  c->launches++;
  const cudaMemcpyKind gkind = gr->mem == KPN_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  const float* red = c->ws_gred.as<float>();
  for (int l = 0; l < NLAYER; ++l) {
    const int nw = (l + 1 < NLAYER ? lay.wo[l + 1] : lay.bo[0]) - lay.wo[l];
    KPN_CUDA(c, cudaMemcpyAsync(gr->dW[l], red + lay.wo[l], (size_t)nw * sizeof(float), gkind, st));
    KPN_CUDA(c, cudaMemcpyAsync(gr->db[l], red + lay.bo[l], (size_t)((l + 1 < NLAYER ? lay.bo[l + 1] : lay.ani) - lay.bo[l]) * sizeof(float),
                                gkind, st));
  }
  KPN_CUDA(c, cudaMemcpyAsync(gr->d_ani_al, red + lay.ani, sizeof(float), gkind, st));
  float* dmaps[3] = {gr->d_feat64, gr->d_feat8, gr->d_feat_tex};
  for (int m = 0; m < 3; ++m) KPN_CUDA(c, cudaMemcpyAsync(dmaps[m], c->ws_gmap[m].p, map_bytes[m], gkind, st));
  return wd_snapshot(c, st);
}

extern "C" int kpn_camera_rays(kpn_ctx* c, const kpn_target* tg, float* origins, float* dirs, float* near_far, int mem, void* stream) {
  if (!c || !tg || !origins || !dirs || !near_far) return KPN_ERR_ARG;
  DeviceGuard g(c->device);
  cudaStream_t st = (cudaStream_t)stream;
  KPN_TRY(check_target(c, tg));
  if (!mem_ok(mem) || !mem_ok(tg->mem)) KPN_FAIL(c, KPN_ERR_ARG, "bad mem kind");
  KPN_TRY(wd_check(c, st));
  const long long R = (long long)tg->nx * tg->ny;
  KPN_TRY(upload_target(c, tg, false, st));
  const float* a[3] = {origins, dirs, near_far};
  const Staging outs = ray_planes(c, false, mem == KPN_MEM_HOST, R, 3, RAY_W, a);
  KPN_TRY(stage(c, outs, st));
  KPN_CUDA(c, launch_camera_rays(c->d_target, 0, R, outs.dev<float>(0), outs.dev<float>(1), outs.dev<float>(2), st));
  c->launches++;
  return unstage(c, outs, st);
}

// The point query shared by kpn_query (query_mode 1: base.pts, base.view) and kpn_query_grid (query_mode 2: the grid of base):
// n points in chunks of 4 Mi, out_w floats per point into out and the validity mask into valid (may be nullptr), both of
// kpn_mem `mem`.  Arguments are checked by the caller.
static int query_points(kpn_ctx* c, const SampleSrc& base, long long n, float* out, int out_w, int query_mode, int mem,
                        uint8_t* valid, const kpn_opts* op, cudaStream_t st) {
  KPN_TRY(begin_counters(c, st));
  if (n == 0) return KPN_OK;
  Staging outs(c, false, mem == KPN_MEM_HOST);
  outs.add(out, (size_t)n * out_w * sizeof(float));
  outs.add(valid, (size_t)n, !valid);   // the compaction writes a mask whether or not the caller wants one
  KPN_TRY(stage(c, outs, st));
  float* dout = outs.dev<float>(0);
  uint8_t* dvalid = outs.dev<uint8_t>(1);
  const long long chunk = 4ll << 20;
  const long long nchunks = (n + chunk - 1) / chunk;
  if (nchunks > MAX_CHUNKS) KPN_FAIL(c, KPN_ERR_ARG, "too many points");
  for (long long ch = 0; ch < nchunks; ++ch) {
    const long long off = ch * chunk;
    const long long m = (n - off) < chunk ? (n - off) : chunk;
    SampleSrc src = base;
    if (query_mode == 1) { src.pts += 3 * off; src.view += 3 * off; }
    else src.g_id0 = off;
    KPN_CUDA(c, c->ws_list.reserve((size_t)m * sizeof(int)));
    KPN_CUDA(c, launch_compact(c->d_scene, src, m, c->ws_list.as<int>(), c->d_counters + ch, dout + out_w * off, out_w, dvalid + off, st));
    c->launches++;
    ShadeOut so;
    memset(&so, 0, sizeof(so));
    (query_mode == 1 ? so.out5 : so.out2) = dout + out_w * off;
    KPN_TRY(shade_batch(c, src, c->ws_list.as<int>(), c->d_counters + ch, c->d_counters2 + ch, m, query_mode, so, op ? op->engine : 0, st));
  }
  c->counters_used = (int)nchunks;
  c->last_total = (unsigned long long)n;
  KPN_TRY(unstage(c, outs, st));
  return wd_snapshot(c, st);
}

extern "C" int kpn_query(kpn_ctx* c, const float* pts, const float* view, int n, float* out5, uint8_t* valid, int mem,
                         const kpn_opts* op, void* stream) {
  if (!c || !pts || !view || !out5 || n < 0) return KPN_ERR_ARG;
  DeviceGuard g(c->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (!c->have_scene) KPN_FAIL(c, KPN_ERR_STATE, "kpn_set_scene must precede kpn_query");
  KPN_TRY(wd_check(c, st));
  if (!mem_ok(mem)) KPN_FAIL(c, KPN_ERR_ARG, "bad mem kind");
  Staging in(c, true, mem == KPN_MEM_HOST);
  in.add(pts, (size_t)n * 3 * sizeof(float));
  in.add(view, (size_t)n * 3 * sizeof(float));
  KPN_TRY(stage(c, in, st));
  SampleSrc src;
  memset(&src, 0, sizeof(src));
  src.mode = 1; src.pts = in.dev<const float>(0); src.view = in.dev<const float>(1);
  return query_points(c, src, n, out5, 5, 1, mem, valid, op, st);
}

extern "C" int kpn_query_grid(kpn_ctx* c, const kpn_grid* g, float* out2, uint8_t* valid, int mem, const kpn_opts* op, void* stream) {
  if (!c || !g || !out2) return KPN_ERR_ARG;
  DeviceGuard dg(c->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (g->nx < 1 || g->ny < 1 || g->nz < 1 || (long long)g->nx * g->ny * g->nz > 0x7fffffffll)
    KPN_FAIL(c, KPN_ERR_ARG, "grid %d x %d x %d: every extent >= 1, at most 2^31 - 1 points", g->nx, g->ny, g->nz);
  for (int a = 0; a < 3; ++a)
    if (!std::isfinite(g->origin[a]) || !std::isfinite(g->spacing[a]) || !(g->spacing[a] > 0.0f))
      KPN_FAIL(c, KPN_ERR_ARG, "grid origin / spacing must be finite, spacing > 0 (axis %d: %g, %g)", a, g->origin[a], g->spacing[a]);
  if (!mem_ok(mem)) KPN_FAIL(c, KPN_ERR_ARG, "bad mem kind");
  if (!c->have_scene) KPN_FAIL(c, KPN_ERR_STATE, "kpn_set_scene must precede kpn_query_grid");
  KPN_TRY(wd_check(c, st));
  SampleSrc src;
  memset(&src, 0, sizeof(src));
  src.mode = 2;
  for (int a = 0; a < 3; ++a) { src.g_org[a] = g->origin[a]; src.g_sp[a] = g->spacing[a]; }
  src.g_nx = g->nx; src.g_ny = g->ny;
  return query_points(c, src, (long long)g->nx * g->ny * g->nz, out2, 2, 2, mem, valid, op, st);
}

// ---------------------------------------------------------------------------------------------
// marching cubes (kpn_mesh.cu)
// ---------------------------------------------------------------------------------------------
extern "C" int kpn_mesh_begin(kpn_ctx* c, const float* field, int nx, int ny, int nz, float level, long long counts[2], void* stream) {
  if (!c || !field || !counts) return KPN_ERR_ARG;
  DeviceGuard dg(c->device);
  cudaStream_t st = (cudaStream_t)stream;
  c->mc_field = nullptr;
  KPN_TRY(wd_check(c, st));
  if (nx < 1 || ny < 1 || nz < 1 || (long long)nx * ny * nz > 0x7fffffffll)
    KPN_FAIL(c, KPN_ERR_ARG, "field %d x %d x %d: every extent >= 1, at most 2^31 - 1 points", nx, ny, nz);
  const int n = nx * ny * nz;
  const long long ncell = (long long)(nx - 1) * (ny - 1) * (nz - 1);
  KPN_CUDA(c, c->mc_vofs.reserve((size_t)n * sizeof(unsigned int)));
  KPN_CUDA(c, c->mc_cases.reserve(ncell > 0 ? (size_t)ncell : 1));
  KPN_CUDA(c, c->mc_tofs.reserve((ncell > 0 ? (size_t)ncell : 1) * sizeof(unsigned int)));
  const size_t scan_bytes = mc_scan_temp_bytes(n);
  KPN_CUDA(c, c->mc_tmp.reserve(scan_bytes));
  KPN_CUDA(c, launch_mc_classify(field, nx, ny, nz, level, c->mc_vofs.as<unsigned int>(), c->mc_cases.as<uint8_t>(),
                                 c->mc_tofs.as<unsigned int>(), c->d_mc_totals, c->mc_tmp.p, scan_bytes, st));
  c->launches += ncell > 0 ? 5 : 3;   // classify + CUB's two kernels per scan
  KPN_CUDA(c, cudaMemcpyAsync(c->h_mc_totals, c->d_mc_totals, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  KPN_CUDA(c, cudaStreamSynchronize(st));
  const unsigned long long nv = c->h_mc_totals[0], nf = c->h_mc_totals[1];
  if (nv > 0x7fffffffull || nf > 0x7fffffffull)
    KPN_FAIL(c, KPN_ERR_ARG, "mesh of %llu vertices, %llu faces: at most 2^31 - 1 of each", nv, nf);
  counts[0] = (long long)nv; counts[1] = (long long)nf;
  c->mc_counts[0] = counts[0]; c->mc_counts[1] = counts[1];
  c->mc_field = field;
  c->mc_dims[0] = nx; c->mc_dims[1] = ny; c->mc_dims[2] = nz;
  c->mc_level = level;
  return KPN_OK;
}

extern "C" int kpn_mesh_emit(kpn_ctx* c, const float* field, const float origin[3], const float spacing[3], float* vertices,
                             float* normals, int* faces, int mem, void* stream) {
  if (!c || !field || !origin || !spacing) return KPN_ERR_ARG;
  DeviceGuard dg(c->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (!mem_ok(mem)) KPN_FAIL(c, KPN_ERR_ARG, "bad mem kind");
  for (int a = 0; a < 3; ++a)
    if (!std::isfinite(origin[a]) || !std::isfinite(spacing[a]) || !(spacing[a] > 0.0f))
      KPN_FAIL(c, KPN_ERR_ARG, "origin / spacing must be finite, spacing > 0 (axis %d: %g, %g)", a, origin[a], spacing[a]);
  if (c->mc_field == nullptr || c->mc_field != field)
    KPN_FAIL(c, KPN_ERR_STATE, "kpn_mesh_begin on the same field must precede kpn_mesh_emit");
  KPN_TRY(wd_check(c, st));
  const long long nv = c->mc_counts[0], nf = c->mc_counts[1];
  if ((nv > 0 && !vertices) || (nf > 0 && !faces)) KPN_FAIL(c, KPN_ERR_ARG, "null vertices / faces for a non-empty mesh");
  Staging outs(c, false, mem == KPN_MEM_HOST);
  outs.add(vertices, (size_t)nv * 3 * sizeof(float));
  outs.add(normals, (size_t)nv * 3 * sizeof(float));
  outs.add(faces, (size_t)nf * 3 * sizeof(int));
  KPN_TRY(stage(c, outs, st));
  KPN_CUDA(c, launch_mc_emit(field, c->mc_dims[0], c->mc_dims[1], c->mc_dims[2], c->mc_level, origin, spacing, c->mc_vofs.as<unsigned int>(),
                             c->mc_cases.as<uint8_t>(), c->mc_tofs.as<unsigned int>(), outs.dev<float>(0), outs.dev<float>(1),
                             outs.dev<int>(2), nf, st));
  c->launches += nf > 0 ? 2 : 1;
  return unstage(c, outs, st);
}

extern "C" int kpn_get_stats(kpn_ctx* c, kpn_stats* stats, void* stream) {
  if (!c || !stats) return KPN_ERR_ARG;
  DeviceGuard g(c->device);
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<int> h(c->counters_used > 0 ? c->counters_used : 1, 0), h2(c->counters_used > 0 ? c->counters_used : 1, 0);
  if (c->counters_used > 0) {
    KPN_CUDA(c, cudaMemcpyAsync(h.data(), c->d_counters, sizeof(int) * c->counters_used, cudaMemcpyDeviceToHost, st));
    KPN_CUDA(c, cudaMemcpyAsync(h2.data(), c->d_counters2, sizeof(int) * c->counters_used, cudaMemcpyDeviceToHost, st));
  }
  KPN_TRY(wd_snapshot(c, st));
  KPN_CUDA(c, cudaStreamSynchronize(st));
  unsigned long long valid = 0, coloured = 0;
  for (int i = 0; i < c->counters_used; ++i) { valid += (unsigned long long)h[i]; coloured += (unsigned long long)h2[i]; }
  stats->samples_total = c->last_total;
  stats->samples_valid = valid;
  stats->samples_coloured = coloured;
  stats->kernel_launches = c->launches;
  double ms = 0.0, gms = 0.0;
  for (size_t i = 0; i + 2 < c->ev_used; i += 3) {   // triples: start, after the geometry kernel, stop
    float t = 0.0f, tg = 0.0f;
    KPN_CUDA(c, cudaEventElapsedTime(&t, c->ev_pool[i], c->ev_pool[i + 2]));
    KPN_CUDA(c, cudaEventElapsedTime(&tg, c->ev_pool[i], c->ev_pool[i + 1]));
    ms += (double)t;
    gms += (double)tg;
  }
  stats->shade_launches = c->ev_used / 3;
  stats->shade_ms = ms;
  stats->geo_ms = gms;
  c->ev_used = 0;
  return wd_check(c, st);
}

// Debug hook.  out16[0..7] receive the device watchdog words of the tensor-core kernels (out16[0] != 0: a barrier wait gave
// up at block out16[1], thread out16[2], tag out16[3]); enable != 0 clears them afterwards.
extern "C" int kpn_debug_timing(kpn_ctx* c, int enable, unsigned long long* out16) {
  if (!c) return KPN_ERR_ARG;
  DeviceGuard g(c->device);
  KPN_CUDA(c, cudaDeviceSynchronize());
  unsigned int wd[TC_WD_MODULES * TC_WD_WORDS];
  KPN_TRY(wd_read(c, wd, nullptr));
  if (enable) KPN_TRY(wd_clear(c, nullptr));
  KPN_CUDA(c, cudaDeviceSynchronize());
  const unsigned int* first = wd[0] != 0u || wd[TC_WD_WORDS] == 0u ? wd : wd + TC_WD_WORDS;   // the first raised module's words
  if (out16) { for (int i = 0; i < 16; ++i) out16[i] = i < 8 ? first[i] : 0ull; }
  return KPN_OK;
}

// Host-only test hook: the K index (element of the fp16 activation row) each input of a geometry stage is multiplied with, and
// the K index of its bias row, for every keypoint count the tensor-core engine covers (tests/test_host_abi.py and
// tests/test_kpt_layout_cpu.py check that the layer-0 permutation is a bijection).
// n_inputs must be the stage's input count (the map is a permutation of exactly those inputs; an index past them has no K row).
extern "C" int kpn_debug_kmap(int stage, int n_kpt, int n_inputs, int* kmap_out, int* kbias_out, int* kpad_out) {
  if (stage < 0 || stage > 5 || !tc_supported(3, n_kpt, 3) || !kmap_out) return KPN_ERR_ARG;
  int dims[NLAYER][2];
  expected_dims(n_kpt, 3, dims);   // geometry stages 0..5 are layers 0..5 (stage 4 also stacks the compress layer, same input)
  if (n_inputs != dims[stage][1]) return KPN_ERR_ARG;
  for (int i = 0; i < n_inputs; ++i) kmap_out[i] = tc_kmap(stage, n_kpt, i);
  if (kbias_out) *kbias_out = tc_kbias(stage, n_kpt);
  if (kpad_out) *kpad_out = make_tc_plan(n_kpt).st[stage].Kp;
  return KPN_OK;
}

// Debug, instrumented build (-DKPN_STAGE_TIMING) only: cycle stamps of one issuer warp of the geometry kernel.  This
// architecture's kernels have no such instrumentation, so every call is refused.
extern "C" int kpn_debug_stage_times(kpn_ctx* c, unsigned long long* out, int n_words, int* n_tiles) {
  if (!c || !out || !n_tiles) return KPN_ERR_ARG;
  KPN_FAIL(c, KPN_ERR_UNSUPPORTED, "library was not built with -DKPN_STAGE_TIMING");
}

extern "C" int kpn_decode_views(kpn_ctx* c, const uint8_t* images, const uint8_t* masks, const double* cams, int n_views, int src_h,
                                int src_w, int factor, float* out_img, uint8_t* out_mask, int mem, void* stream) {
  if (!c || !images || !cams || !out_img) return KPN_ERR_ARG;
  DeviceGuard g(c->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (n_views < 1 || src_h < 1 || src_w < 1 || factor < 1 || src_h % factor || src_w % factor)
    KPN_FAIL(c, KPN_ERR_ARG, "decode: %d views of %dx%d by 1/%d", n_views, src_h, src_w, factor);
  if (!mem_ok(mem)) KPN_FAIL(c, KPN_ERR_ARG, "bad mem kind");
  const size_t npx = (size_t)n_views * src_h * src_w, nout = npx / ((size_t)factor * factor);
  Staging in(c, true, mem == KPN_MEM_HOST), outs(c, false, mem == KPN_MEM_HOST);
  in.add(cams, (size_t)n_views * 18 * sizeof(double));
  in.add(images, npx * 3);
  in.add(masks, npx);
  outs.add(out_img, nout * 3 * sizeof(float));
  outs.add(out_mask, nout);
  KPN_TRY(stage(c, in, st));
  KPN_TRY(stage(c, outs, st));
  KPN_CUDA(c, launch_decode_views(in.dev<const uint8_t>(1), in.dev<const uint8_t>(2), in.dev<const void>(0), n_views, src_h, src_w,
                                  factor, outs.dev<float>(0), outs.dev<uint8_t>(1), st));
  c->launches++;
  return unstage(c, outs, st);
}

extern "C" int kpn_set_profiling(kpn_ctx* c, int enable) {
  if (!c) return KPN_ERR_ARG;
  c->profiling = enable != 0;
  return KPN_OK;
}
