// Source-view decode on the device (SURVEY.md section 8f.4): what ZJUDataset.__getitem__ does to every view on CPU workers
// (reference src/zju_dataset.py:266-287) as ONE kernel:
//   cv2.undistort(image float32 / 255, K, D) and cv2.undistort(mask uint8, K, D)   (bilinear remap, BORDER_CONSTANT 0)
//   cv2.resize(image, ratio, INTER_AREA) / cv2.resize(mask, ratio, INTER_NEAREST)    (ratio = 1 / factor, factor integer)
//   image[mask == 0] = 0 ; mask = mask != 0 ; image -> (3, H, W)
// The arithmetic restates OpenCV's so that the result is bit-identical to the reference's (tests/test_gpu_decode.py compares
// with the cv2 calls themselves):
//   * undistort map per DESTINATION pixel in double precision: (x, y) = K^-1 (u, v, 1), radial/tangential distortion
//     (k1, k2, p1, p2, k3), back through K; coordinates are quantised to 1/32 pixel (cvRound(u * 32), round-half-even);
//   * float image: taps weighted (1-fx)(1-fy), fx(1-fy), (1-fx)fy, fx*fy with fx, fy multiples of 1/32, summed left to right in
//     fp32 without fused multiply-adds; taps outside the image contribute 0;
//   * uint8 mask: the same weights in 15-bit fixed point (exact for multiples of 1/32), (sum + 2^14) >> 15;
//   * INTER_AREA with an integer factor is the box average: the factor^2 taps in row-major order, summed four at a time
//     (((t0 + t1) + t2) + t3 added to the running sum, OpenCV's unrolled loop; the remainder one by one), times 1 / factor^2 in
//     fp32; INTER_NEAREST takes the top-left source pixel of each box.
// HBM-bound byte work: 3 bytes in and 12 + 1 bytes out per output pixel times factor^2 taps; no tensor cores involved.
#include <stdint.h>
#include "kpn_launch.h"

namespace kpn {

struct DecodeView {
  double ir[9];                   // inverse of the 3x3 camera matrix
  double fx, fy, cx, cy, k1, k2, p1, p2, k3;
};

__device__ __forceinline__ void undistort_src(const DecodeView& c, int u, int v, int& sx, int& sy, int& a, int& b) {
  // (no FMA contraction in this function: the products and sums round like OpenCV's scalar code)
  const double du = (double)u, dv = (double)v;
  const double X = __dadd_rn(__dadd_rn(__dmul_rn(du, c.ir[0]), __dmul_rn(dv, c.ir[1])), c.ir[2]);
  const double Y = __dadd_rn(__dadd_rn(__dmul_rn(du, c.ir[3]), __dmul_rn(dv, c.ir[4])), c.ir[5]);
  const double W = __dadd_rn(__dadd_rn(__dmul_rn(du, c.ir[6]), __dmul_rn(dv, c.ir[7])), c.ir[8]);
  const double x = __ddiv_rn(X, W), y = __ddiv_rn(Y, W);
  const double x2 = __dmul_rn(x, x), y2 = __dmul_rn(y, y), r2 = __dadd_rn(x2, y2), xy2 = __dmul_rn(__dmul_rn(2.0, x), y);
  const double kr = __dadd_rn(1.0, __dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(c.k3, r2), c.k2), r2), c.k1), r2));
  const double xd = __dadd_rn(__dadd_rn(__dmul_rn(x, kr), __dmul_rn(c.p1, xy2)), __dmul_rn(c.p2, __dadd_rn(r2, __dmul_rn(2.0, x2))));
  const double yd = __dadd_rn(__dadd_rn(__dmul_rn(y, kr), __dmul_rn(c.p1, __dadd_rn(r2, __dmul_rn(2.0, y2)))), __dmul_rn(c.p2, xy2));
  const double us = __dadd_rn(__dmul_rn(c.fx, xd), c.cx), vs = __dadd_rn(__dmul_rn(c.fy, yd), c.cy);
  const long long iu = __double2ll_rn(__dmul_rn(us, 32.0)), iv = __double2ll_rn(__dmul_rn(vs, 32.0));   // cvRound: half to even
  sx = (int)(iu >> 5); sy = (int)(iv >> 5); a = (int)(iu & 31); b = (int)(iv & 31);
}

__global__ void __launch_bounds__(256)
decode_views_kernel(const uint8_t* __restrict__ images, const uint8_t* __restrict__ masks, const DecodeView* __restrict__ cams,
                    int V, int H0, int W0, int factor, float* __restrict__ out_img, uint8_t* __restrict__ out_mask) {
  const int H = H0 / factor, W = W0 / factor;
  const long long n = (long long)V * H * W;
  const float inv_area = 1.0f / (float)(factor * factor);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W), y = (int)((i / W) % H), v = (int)(i / ((long long)W * H));
    const DecodeView& c = cams[v];
    const uint8_t* im = images + (size_t)v * H0 * W0 * 3;
    const uint8_t* mk = masks ? masks + (size_t)v * H0 * W0 : nullptr;
    float acc[3] = {0.0f, 0.0f, 0.0f}, grp[3] = {0.0f, 0.0f, 0.0f};
    const int area = factor * factor, nfull = area & ~3;
    int fg = 1, k = 0;
    for (int dy = 0; dy < factor; ++dy)
      for (int dx = 0; dx < factor; ++dx, ++k) {
        int sx, sy, a, b;
        undistort_src(c, x * factor + dx, y * factor + dy, sx, sy, a, b);
        const float fx = (float)a * (1.0f / 32.0f), fy = (float)b * (1.0f / 32.0f);
        const float w[4] = {__fmul_rn(1.0f - fx, 1.0f - fy), __fmul_rn(fx, 1.0f - fy), __fmul_rn(1.0f - fx, fy), __fmul_rn(fx, fy)};
        const int xs[4] = {sx, sx + 1, sx, sx + 1}, ys[4] = {sy, sy, sy + 1, sy + 1};
        float px[3] = {0.0f, 0.0f, 0.0f};
        int msum = 0;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const bool in = xs[t] >= 0 && xs[t] < W0 && ys[t] >= 0 && ys[t] < H0;
          const size_t o = in ? (size_t)ys[t] * W0 + xs[t] : 0;
#pragma unroll
          for (int ch = 0; ch < 3; ++ch) {
            const float p = in ? __fdiv_rn((float)im[3 * o + ch], 255.0f) : 0.0f;   // imread(...).astype(float32) / 255.
            px[ch] = t == 0 ? __fmul_rn(p, w[0]) : __fadd_rn(px[ch], __fmul_rn(p, w[t]));
          }
          if (dy == 0 && dx == 0 && mk) {
            const int wi = (t == 0 ? (32 - a) * (32 - b) : t == 1 ? a * (32 - b) : t == 2 ? (32 - a) * b : a * b) * 32;
            msum += (in && mk[o] != 0 ? 1 : 0) * wi;
          }
        }
        if (dy == 0 && dx == 0 && mk) fg = ((msum + (1 << 14)) >> 15) != 0;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
          if (k < nfull) {
            grp[ch] = (k & 3) == 0 ? px[ch] : __fadd_rn(grp[ch], px[ch]);
            if ((k & 3) == 3) acc[ch] = __fadd_rn(acc[ch], grp[ch]);
          } else {
            acc[ch] = __fadd_rn(acc[ch], px[ch]);
          }
        }
      }
    const size_t plane = (size_t)H * W, o = (size_t)y * W + x;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch)
      out_img[((size_t)v * 3 + ch) * plane + o] = fg ? (factor > 1 ? __fmul_rn(acc[ch], inv_area) : acc[ch]) : 0.0f;
    if (out_mask) out_mask[(size_t)v * plane + o] = (uint8_t)fg;
  }
}

cudaError_t launch_decode_views(const uint8_t* images, const uint8_t* masks, const void* cams, int V, int H0, int W0, int factor,
                                float* out_img, uint8_t* out_mask, cudaStream_t st) {
  const long long n = (long long)V * (H0 / factor) * (W0 / factor);
  long long g = (n + 255) / 256;
  if (g > 132 * 16) g = 132 * 16;
  if (g < 1) g = 1;
  decode_views_kernel<<<(int)g, 256, 0, st>>>(images, masks, reinterpret_cast<const DecodeView*>(cams), V, H0, W0, factor, out_img, out_mask);
  return cudaGetLastError();
}

}  // namespace kpn
