// The parts of LPIPS (vidtok/modules/lpips.py) around its VGG16 convolutions: the 2x2 max-pools between the slices and the
// per-position head of each tap, on the channels-last bf16 / hi|lo split activations the convolutions write.  The
// convolutions themselves are conv_tc launches with the ReLU epilogue, and conv1_1 is the LPIPS stem of conv_stem.cu.
//
// Head (lpips.py:82-95,166-172): per position of tap k, f / (sqrt(sum_c f^2) + 1e-10) for the two images, the squared
// difference, then lin_k (a 1 x 1 convolution to one channel without bias), then the mean over H_k x W_k; LPIPS is the sum
// of the five layers' means.  One CTA takes kLpipsHeadPos positions of one image pair and writes their sum (fp32) to the
// workspace; the finish kernel adds an image's partials in index order in double.  No atomics: the same input gives the
// same bits, whatever the stream or the pass the frame falls into.
#include <cstdio>

#include "common.cuh"
#include "kernels.h"

namespace vt {
namespace {

constexpr int kThreads = 256;

// 8 consecutive 16-bit channels as floats; split: hi + lo (the lo plane C elements further)
template <bool kSplit>
__device__ __forceinline__ void load8(const bf16* p, int C, float (&v)[8], uint4& hw, uint4& lw) {
  hw = *reinterpret_cast<const uint4*>(p);
  const uint32_t* h = reinterpret_cast<const uint32_t*>(&hw);
  if constexpr (kSplit) {
    lw = *reinterpret_cast<const uint4*>(p + C);
    const uint32_t* l = reinterpret_cast<const uint32_t*>(&lw);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&h[e]));
      const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&l[e]));
      v[2 * e] = a.x + b.x;
      v[2 * e + 1] = a.y + b.y;
    }
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&h[e]));
      v[2 * e] = a.x;
      v[2 * e + 1] = a.y;
    }
  }
}

// One thread per output position and 8 channels.  torch's max_pool2d: the first maximum of the window wins, a NaN wins.
template <bool kSplit>
__global__ void __launch_bounds__(kThreads) maxpool2x2_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, long long total, int H,
                                                             int W, int Ho, int Wo, int C) {
  const int U = C / 8;
  const long long cs = kSplit ? 2LL * C : (long long)C;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
    const int u = (int)(i % U);
    long long r = i / U;
    const int wo = (int)(r % Wo);
    r /= Wo;
    const int ho = (int)(r % Ho);
    const long long n = r / Ho;
    const bf16* src = x + ((n * H + 2 * ho) * W + 2 * wo) * cs + 8 * u;
    float best[8], v[8];
    uint4 bh, bl, h, l;
    load8<kSplit>(src, C, best, bh, bl);
    uint16_t* bhs = reinterpret_cast<uint16_t*>(&bh);
    uint16_t* bls = reinterpret_cast<uint16_t*>(&bl);
#pragma unroll
    for (int q = 1; q < 4; ++q) {
      load8<kSplit>(src + ((q >> 1) * (long long)W + (q & 1)) * cs, C, v, h, l);
      const uint16_t* hs = reinterpret_cast<const uint16_t*>(&h);
      const uint16_t* ls = reinterpret_cast<const uint16_t*>(&l);
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (v[e] > best[e] || v[e] != v[e]) {
          best[e] = v[e];
          bhs[e] = hs[e];
          if constexpr (kSplit) bls[e] = ls[e];
        }
    }
    bf16* dst = y + ((n * Ho + ho) * Wo + wo) * cs + 8 * u;
    *reinterpret_cast<uint4*>(dst) = bh;
    if constexpr (kSplit) *reinterpret_cast<uint4*>(dst + C) = bl;
  }
}

// The max-pools of I3D (metrics FVD): window kt x kh x kw, strides st x sh x sw, front padding pt, ph, pw ("SAME"), over
// channels-last [N,T,H,W,C] (split: [.., hi C | lo C], compared as hi + lo) -> [N,To,Ho,Wo,C].  A padded position counts as a
// zero, which is what ignoring it gives on the ReLU outputs this pools.  Window order (t, h, w); the first maximum wins, a
// NaN wins.
template <bool kSplit>
__global__ void __launch_bounds__(kThreads) maxpool3d_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, long long total, MaxPool3d q) {
  const int U = q.C / 8;
  const long long cs = kSplit ? 2LL * q.C : (long long)q.C;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
    const int u = (int)(i % U);
    long long r = i / U;
    const int wo = (int)(r % q.Wo);
    r /= q.Wo;
    const int ho = (int)(r % q.Ho);
    r /= q.Ho;
    const int to = (int)(r % q.To);
    const long long n = r / q.To;
    float best[8], v[8];
    uint4 bh = make_uint4(0, 0, 0, 0), bl = make_uint4(0, 0, 0, 0), h, l;
#pragma unroll
    for (int e = 0; e < 8; ++e) best[e] = -INFINITY;
    uint16_t* bhs = reinterpret_cast<uint16_t*>(&bh);
    uint16_t* bls = reinterpret_cast<uint16_t*>(&bl);
    for (int a = 0; a < q.kt; ++a)
      for (int b = 0; b < q.kh; ++b)
        for (int c = 0; c < q.kw; ++c) {
          const int ti = to * q.st + a - q.pt, hi = ho * q.sh + b - q.ph, wi = wo * q.sw + c - q.pw;
          if (ti >= 0 && ti < q.T && hi >= 0 && hi < q.H && wi >= 0 && wi < q.W) {
            load8<kSplit>(x + (((n * q.T + ti) * q.H + hi) * q.W + wi) * cs + 8 * u, q.C, v, h, l);
          } else {
            h = l = make_uint4(0, 0, 0, 0);
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = 0.f;
          }
          const uint16_t* hs = reinterpret_cast<const uint16_t*>(&h);
          const uint16_t* ls = reinterpret_cast<const uint16_t*>(&l);
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (v[e] > best[e] || v[e] != v[e]) {
              best[e] = v[e];
              bhs[e] = hs[e];
              if constexpr (kSplit) bls[e] = ls[e];
            }
        }
    bf16* dst = y + (((n * q.To + to) * q.Ho + ho) * q.Wo + wo) * cs + 8 * u;
    *reinterpret_cast<uint4*>(dst) = bh;
    if constexpr (kSplit) *reinterpret_cast<uint4*>(dst + q.C) = bl;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
  // xor butterfly: every lane ends with the same value (fp addition is commutative)
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
  return v;
}

// channel pair (c, c + 1) of a position; split: hi + lo
template <bool kSplit>
__device__ __forceinline__ float2 load2(const bf16* p, int C, int c) {
  const uint32_t hw = *reinterpret_cast<const uint32_t*>(p + c);
  if constexpr (kSplit) {
    const uint32_t lw = *reinterpret_cast<const uint32_t*>(p + C + c);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&hw));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&lw));
    return make_float2(a.x + b.x, a.y + b.y);
  } else {
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hw));
  }
}

// Block (g, tile): warp wq takes positions [tile * kLpipsHeadPos + wq * kPerWarp, +kPerWarp) of image pair g, lane l the channel
// pairs 2 l, 2 l + 64, ...; the warp's positions are added in order, then the warps in order.
template <bool kSplit>
__global__ void __launch_bounds__(kThreads) lpips_head_kernel(const bf16* __restrict__ f, int G, long long HW, int C, const float* __restrict__ w,
                                                             float* __restrict__ part, long long tiles) {
  constexpr int kPerWarp = kLpipsHeadPos / (kThreads / 32);
  __shared__ float red[kThreads / 32];
  const long long g = blockIdx.x / tiles, tile = blockIdx.x % tiles;
  const int wq = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long cs = kSplit ? 2LL * C : (long long)C;
  const bf16* fx = f + g * HW * cs;
  const bf16* fy = f + (G + g) * HW * cs;
  float acc = 0.f;
  for (int k = 0; k < kPerWarp; ++k) {
    const long long pos = tile * kLpipsHeadPos + wq * kPerWarp + k;
    if (pos >= HW) break;
    const bf16* px = fx + pos * cs;
    const bf16* py = fy + pos * cs;
    float sx = 0.f, sy = 0.f;
    for (int c = 2 * lane; c < C; c += 64) {
      const float2 a = load2<kSplit>(px, C, c), b = load2<kSplit>(py, C, c);
      sx = fmaf(a.x, a.x, sx); sx = fmaf(a.y, a.y, sx);
      sy = fmaf(b.x, b.x, sy); sy = fmaf(b.y, b.y, sy);
    }
    const float nx = __fadd_rn(sqrtf(warp_sum(sx)), 1e-10f), ny = __fadd_rn(sqrtf(warp_sum(sy)), 1e-10f);
    float d = 0.f;
    for (int c = 2 * lane; c < C; c += 64) {
      const float2 a = load2<kSplit>(px, C, c), b = load2<kSplit>(py, C, c);
      const float d0 = __fsub_rn(__fdiv_rn(a.x, nx), __fdiv_rn(b.x, ny));
      const float d1 = __fsub_rn(__fdiv_rn(a.y, nx), __fdiv_rn(b.y, ny));
      d = fmaf(w[c], __fmul_rn(d0, d0), d);
      d = fmaf(w[c + 1], __fmul_rn(d1, d1), d);
    }
    acc += warp_sum(d);
  }
  if (lane == 0) red[wq] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < kThreads / 32; ++i) s += red[i];
    part[g * tiles + tile] = s;
  }
}

__global__ void __launch_bounds__(kThreads) lpips_finish_kernel(const float* __restrict__ part, LpipsFinish fin, int G, float* __restrict__ lpips,
                                                               float* __restrict__ per_layer, double* __restrict__ running) {
  for (int g = threadIdx.x; g < G; g += kThreads) {
    double total = 0.0;
    for (int k = 0; k < 5; ++k) {
      const float* p = part + fin.off[k] + (long long)g * fin.tiles[k];
      double s = 0.0;
      for (long long i = 0; i < fin.tiles[k]; ++i) s += (double)p[i];
      const double r = s / fin.area[k];
      if (per_layer) per_layer[(long long)g * 5 + k] = (float)r;
      total += r;
    }
    lpips[g] = (float)total;
  }
  __syncthreads();
  if (running && threadIdx.x == 0) {
    double s = running[0];
    for (int g = 0; g < G; ++g) s += (double)lpips[g];
    running[0] = s;
    running[1] += (double)G;
  }
}

unsigned grid_for(long long work) {
  long long g = (work + kThreads - 1) / kThreads;
  if (g > 132 * 16) g = 132 * 16;
  return (unsigned)(g < 1 ? 1 : g);
}

}  // namespace

cudaError_t launch_maxpool2x2(const bf16* x, bf16* y, long long N, int H, int W, int C, bool split, cudaStream_t s) {
  if (C % 8 != 0 || H < 2 || W < 2) return cudaErrorInvalidValue;
  const int Ho = H / 2, Wo = W / 2;
  const long long total = N * Ho * Wo * (C / 8);
  const double esz = split ? 4.0 : 2.0;
  char det[64] = "";
  if (prof_enabled()) snprintf(det, sizeof(det), "%lldx%dx%dx%d%s", N, H, W, C, split ? " split" : "");
  ProfScope _ps("maxpool2x2", 3.0 * N * Ho * Wo * C, esz * ((double)N * H * W * C + (double)N * Ho * Wo * C), s, det);
  if (split) maxpool2x2_kernel<true><<<grid_for(total), kThreads, 0, s>>>(x, y, total, H, W, Ho, Wo, C);
  else maxpool2x2_kernel<false><<<grid_for(total), kThreads, 0, s>>>(x, y, total, H, W, Ho, Wo, C);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_maxpool3d(const bf16* x, bf16* y, long long N, const MaxPool3d& q, bool split, cudaStream_t s) {
  if (q.C % 8 != 0 || q.To < 1 || q.Ho < 1 || q.Wo < 1) return cudaErrorInvalidValue;
  const long long total = N * q.To * q.Ho * q.Wo * (q.C / 8);
  const double esz = split ? 4.0 : 2.0, out = (double)N * q.To * q.Ho * q.Wo * q.C;
  char det[96] = "";
  if (prof_enabled()) snprintf(det, sizeof(det), "k%d%d%d s%d%d%d %lldx%dx%dx%dx%d%s", q.kt, q.kh, q.kw, q.st, q.sh, q.sw, N, q.T, q.H, q.W, q.C, split ? " split" : "");
  ProfScope _ps("maxpool3d", out * q.kt * q.kh * q.kw, esz * ((double)N * q.T * q.H * q.W * q.C + out), s, det);
  if (split) maxpool3d_kernel<true><<<grid_for(total), kThreads, 0, s>>>(x, y, total, q);
  else maxpool3d_kernel<false><<<grid_for(total), kThreads, 0, s>>>(x, y, total, q);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_lpips_head(const bf16* f, int G, int H, int W, int C, bool split, const float* w, float* part, cudaStream_t s) {
  if (C % 64 != 0) return cudaErrorInvalidValue;
  const long long HW = (long long)H * W, tiles = lpips_head_tiles(H, W);
  const double esz = split ? 4.0 : 2.0;
  char det[64] = "";
  if (prof_enabled()) snprintf(det, sizeof(det), "%dx%dx%dx%d%s", 2 * G, H, W, C, split ? " split" : "");
  // per position and channel: two squares, two divisions, a difference, its square and the weighted sum for the pair
  ProfScope _ps("lpips_head", (double)G * HW * C * 8.0, esz * 2.0 * G * HW * C + (double)G * tiles * 4.0, s, det);
  const unsigned grid = (unsigned)((long long)G * tiles);
  if (split) lpips_head_kernel<true><<<grid, kThreads, 0, s>>>(f, G, HW, C, w, part, tiles);
  else lpips_head_kernel<false><<<grid, kThreads, 0, s>>>(f, G, HW, C, w, part, tiles);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_lpips_finish(const float* part, const LpipsFinish& f, int G, float* lpips, float* per_layer, double* running,
                                cudaStream_t s) {
  double parts = 0.0;
  for (int k = 0; k < 5; ++k) parts += (double)G * f.tiles[k];
  ProfScope _ps("lpips_finish", parts, parts * 4.0 + G * 4.0 * (per_layer ? 6.0 : 1.0), s);
  lpips_finish_kernel<<<1, kThreads, 0, s>>>(part, f, G, lpips, per_layer, running);
  count_launch();
  return cudaGetLastError();
}

}  // namespace vt
