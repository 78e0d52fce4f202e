// Resize -> CenterCrop -> Normalize of decoded uint8 frames in one launch (vt_video_u8_to_clip_resized): the transform the
// reference applies to every clip (scripts/inference_reconstruct.py:41-47,73-74, vidtok/data/vidtok.py:51-56,181-185):
//   Resize(short side, antialias=True) -> CenterCrop((H, W)) -> Normalize(.5, .5) on frames.float() / 255.
// The Resize is torch's CPU _upsample_bilinear2d_aa (align_corners=False), restated operation by operation so that the
// result is the CPU result bit for bit: taps and weights with torch's mix of float and double, the W pass before the H
// pass, and the per-output tap sum in the order and with the rounding torch's compiled CPU loop uses (see tap_sum).
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "kernels.h"

namespace vt {
namespace {

constexpr int kThreads = 256;
constexpr size_t kSmemMax = 227 * 1024;
constexpr int kTiles[] = {16, 8, 4, 2, 1};   // output tile side, largest first

// One dimension of the antialiased bilinear resize, in torch's types: scale = in/out in float, support = scale for a
// downscale and 1 (plain bilinear) otherwise, taps per output at most ceil(support)*2+1.
struct AaAxis {
  int in;
  float scale, support, invscale;
  int K;
};

AaAxis make_axis(int in, int out) {
  AaAxis a;
  a.in = in;
  a.scale = (float)in / (float)out;
  a.support = a.scale >= 1.0f ? (float)(1.0 * (double)a.scale) : 1.0f;
  a.invscale = a.scale >= 1.0f ? (float)(1.0 / (double)a.scale) : 1.0f;
  a.K = (int)std::ceil(a.support) * 2 + 1;
  return a;
}

// First source index and tap count of output index i (center in float from a double product, bounds in double).
__host__ __device__ inline void aa_bounds(const AaAxis& a, int i, float& center, int& lo, int& n) {
  center = (float)((double)a.scale * ((double)i + 0.5));
  long long x0 = (long long)((double)(center - a.support) + 0.5);
  long long x1 = (long long)((double)(center + a.support) + 0.5);
  x0 = x0 < 0 ? 0 : x0;
  x1 = x1 > a.in ? a.in : x1;
  long long m = x1 - x0;
  lo = (int)x0;
  n = (int)(m < 0 ? 0 : (m > a.K ? a.K : m));
}

// Normalised triangle-filter weights of output index i: filter((j + lo - center + 0.5) * invscale), summed and divided in
// float.  The argument is rounded once from double, as torch passes a double expression to a float filter.
__device__ inline void aa_taps(const AaAxis& a, int i, int& lo, int& n, float* w) {
  float center;
  aa_bounds(a, i, center, lo, n);
  float total = 0.0f;
  for (int j = 0; j < n; ++j) {
    const float d = __fsub_rn((float)(j + lo), center);
    const float x = fabsf(__double2float_rn(__dmul_rn(__dadd_rn((double)d, 0.5), (double)a.invscale)));
    w[j] = x < 1.0f ? __fsub_rn(1.0f, x) : 0.0f;
    total = __fadd_rn(total, w[j]);
  }
  if (total != 0.0f)
    for (int j = 0; j < n; ++j) w[j] = __fdiv_rn(w[j], total);
}

// The tap sum of torch's CPU loop (output = t0*w0; output += tj*wj) as its x86 build evaluates it: the taps after the
// first go in groups of four through a vectorised in-order reduction (product rounded, then added), and the remaining
// (n-1) % 4 taps through scalar FMA.  Other CPU builds may contract differently; the sum order is the same.
template <typename Tap>
__device__ inline float tap_sum(Tap v, const float* w, int n) {
  float acc = __fmul_rn(v(0), w[0]);
  const int grouped = 1 + ((n - 1) / 4) * 4;
  int j = 1;
  for (; j < grouped; ++j) acc = __fadd_rn(acc, __fmul_rn(v(j), w[j]));
  for (; j < n; ++j) acc = __fmaf_rn(v(j), w[j], acc);
  return acc;
}

struct Plan {
  int T;                   // output tile side
  int rows, cols;          // largest source window of one tile
  int pitch;               // staged bytes per window row (room for the 0-3 byte word-alignment shift)
  size_t off_w, off_tmp, off_src, smem;
};

// Largest source window, in source indices, that one tile of T consecutive outputs of [off, off+len) reads.
int max_window(const AaAxis& a, int off, int len, int T) {
  int best = 0;
  for (int t0 = 0; t0 < len; t0 += T) {
    int lo = 1 << 30, hi = 0;
    for (int i = t0; i < std::min(len, t0 + T); ++i) {
      float c;
      int l, n;
      aa_bounds(a, off + i, c, l, n);
      lo = std::min(lo, l);
      hi = std::max(hi, l + n);
    }
    best = std::max(best, hi - lo);
  }
  return best;
}

__host__ __device__ inline size_t up16(size_t b) { return (b + 15) & ~(size_t)15; }

Plan make_plan(const AaAxis& ay, const AaAxis& ax, int h0, int w0, int H, int W, int C, int T) {
  Plan p;
  p.T = T;
  p.rows = max_window(ay, h0, H, T);
  p.cols = max_window(ax, w0, W, T);
  p.pitch = (int)((p.cols * C + 3 + 3) & ~3);
  p.off_w = up16(256 * sizeof(float)) + up16(4 * T * sizeof(int));
  p.off_tmp = p.off_w + up16((size_t)T * (ax.K + ay.K) * sizeof(float));
  p.off_src = p.off_tmp + up16((size_t)p.rows * T * C * sizeof(float));
  p.smem = p.off_src + (size_t)p.rows * p.pitch;
  return p;
}

__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(gmem) : "memory");
}

// One CTA: one T x T tile of the crop of one frame, all channels.  It computes its taps, stages the uint8 source window in
// shared memory, runs the W pass over every window row into fp32 shared memory, then the H pass straight to the clip.
__global__ void __launch_bounds__(kThreads) u8_frames_resize_to_clip_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst,
                                                                           int Hs, int Ws, int C, AaAxis ay, AaAxis ax, int h0, int w0,
                                                                           int H, int W, int Tc, Plan p, int tiles_w, int tiles) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int T = p.T;
  float* lut = reinterpret_cast<float*>(smem);
  int* xlo = reinterpret_cast<int*>(smem + up16(256 * sizeof(float)));
  int* xn = xlo + T;
  int* ylo = xn + T;
  int* yn = ylo + T;
  float* wx = reinterpret_cast<float*>(smem + p.off_w);
  float* wy = wx + T * ax.K;
  float* tmp = reinterpret_cast<float*>(smem + p.off_tmp);
  unsigned char* stage = smem + p.off_src;

  const int n = blockIdx.x / tiles;
  const int tile = blockIdx.x % tiles;
  const int ty0 = (tile / tiles_w) * T, tx0 = (tile % tiles_w) * T;
  const int th = min(T, H - ty0), tw = min(T, W - tx0);
  const int tid = threadIdx.x;

  for (int i = tid; i < 256; i += kThreads) lut[i] = __fdiv_rn((float)i, 255.0f);   // frames.float() / 255.0
  if (tid < tw) aa_taps(ax, w0 + tx0 + tid, xlo[tid], xn[tid], wx + tid * ax.K);
  else if (tid >= T && tid < T + th) aa_taps(ay, h0 + ty0 + tid - T, ylo[tid - T], yn[tid - T], wy + (tid - T) * ay.K);
  __syncthreads();

  int c0 = xlo[0], c1 = 0, r0 = ylo[0], r1 = 0;
  for (int i = 0; i < tw; ++i) { c0 = min(c0, xlo[i]); c1 = max(c1, xlo[i] + xn[i]); }
  for (int i = 0; i < th; ++i) { r0 = min(r0, ylo[i]); r1 = max(r1, ylo[i] + yn[i]); }
  const int nr = r1 - r0, len = (c1 - c0) * C;

  // Stage: each window row is `len` contiguous bytes of the HWC frame.  Staged row byte k holds global byte
  // (row start & ~3) + k, so whole aligned words go through 4-byte cp.async and only the partial end words bytewise.
  const uint8_t* frame = src + (long long)n * Hs * Ws * C;
  const int wpr = (len + 6) / 4;
  for (int q = tid; q < nr * wpr; q += kThreads) {
    const int r = q / wpr, u = q % wpr;
    const uint8_t* g = frame + ((long long)(r0 + r) * Ws + c0) * C;
    const int sh = (int)((uintptr_t)g & 3);
    const int b0 = 4 * u - sh;   // first byte of this word, relative to g
    if (b0 >= len || b0 + 4 <= 0) continue;
    unsigned char* s = stage + r * p.pitch + 4 * u;
    if (b0 >= 0 && b0 + 4 <= len) cp_async4(s, g + b0);
    else
      for (int k = 0; k < 4; ++k)
        if (b0 + k >= 0 && b0 + k < len) s[k] = g[b0 + k];
  }
  asm volatile("cp.async.wait_all;\n" ::: "memory");
  __syncthreads();

  // W pass: tmp[r][x][c] for every window row
  const int twc = tw * C;
  for (int q = tid; q < nr * twc; q += kThreads) {
    const int r = q / twc, xc = q % twc;
    const int x = xc / C, c = xc % C;
    const uint8_t* g = frame + ((long long)(r0 + r) * Ws + c0) * C;
    const unsigned char* s = stage + r * p.pitch + ((uintptr_t)g & 3) + (xlo[x] - c0) * C + c;
    tmp[r * T * C + xc] = tap_sum([&](int j) { return lut[s[j * C]]; }, wx + x * ax.K, xn[x]);
  }
  __syncthreads();

  // H pass and Normalize: clip [N/Tc, C, Tc, H, W], x fastest for coalesced stores
  const int clip = n / Tc, t = n % Tc;
  for (int q = tid; q < th * tw * C; q += kThreads) {
    const int x = q % tw, y = (q / tw) % th, c = q / (tw * th);
    const float* v = tmp + (ylo[y] - r0) * T * C + x * C + c;
    const float acc = tap_sum([&](int j) { return v[j * T * C]; }, wy + y * ay.K, yn[y]);
    dst[(((long long)(clip * C + c) * Tc + t) * H + ty0 + y) * W + tx0 + x] = __fdiv_rn(__fsub_rn(acc, 0.5f), 0.5f);
  }
}

bool plan_for(int Hs, int Ws, int C, int Hr, int Wr, int h0, int w0, int H, int W, AaAxis& ay, AaAxis& ax, Plan& p) {
  ay = make_axis(Hs, Hr);
  ax = make_axis(Ws, Wr);
  for (int T : kTiles) {
    p = make_plan(ay, ax, h0, w0, H, W, C, T);
    if (p.smem <= kSmemMax) return true;
  }
  return false;
}

}  // namespace

bool u8_frames_resize_fits(int Hs, int Ws, int C, int Hr, int Wr, int h0, int w0, int H, int W) {
  AaAxis ay, ax;
  Plan p;
  return plan_for(Hs, Ws, C, Hr, Wr, h0, w0, H, W, ay, ax, p);
}

cudaError_t launch_u8_frames_resize_to_clip(const uint8_t* src, float* dst, int N, int Hs, int Ws, int C, int Hr, int Wr, int h0,
                                            int w0, int H, int W, int Tc, cudaStream_t s) {
  AaAxis ay, ax;
  Plan p;
  if (!plan_for(Hs, Ws, C, Hr, Wr, h0, w0, H, W, ay, ax, p)) return cudaErrorInvalidValue;
  // algorithmic bytes: the source rectangle the crop's taps cover, read once, and the fp32 clip written once
  float cf;
  int ylo0, yn0, ylo1, yn1, xlo0, xn0, xlo1, xn1;
  aa_bounds(ay, h0, cf, ylo0, yn0);
  aa_bounds(ay, h0 + H - 1, cf, ylo1, yn1);
  aa_bounds(ax, w0, cf, xlo0, xn0);
  aa_bounds(ax, w0 + W - 1, cf, xlo1, xn1);
  const double bytes = (double)N * C * ((double)(ylo1 + yn1 - ylo0) * (xlo1 + xn1 - xlo0) + 4.0 * H * W);
  ProfScope _ps("u8_frames_resize_to_clip", 0.0, bytes, s);
  cudaError_t e = cudaFuncSetAttribute(u8_frames_resize_to_clip_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemMax);
  if (e != cudaSuccess) return e;
  const int tiles_w = (W + p.T - 1) / p.T, tiles = tiles_w * ((H + p.T - 1) / p.T);
  u8_frames_resize_to_clip_kernel<<<(unsigned)((long long)N * tiles), kThreads, p.smem, s>>>(src, dst, Hs, Ws, C, ay, ax, h0, w0, H, W,
                                                                                            Tc, p, tiles_w, tiles);
  count_launch();
  return cudaGetLastError();
}

}  // namespace vt
