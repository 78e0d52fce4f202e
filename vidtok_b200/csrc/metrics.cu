// Per-frame PSNR and SSIM of a reconstruction against its input in one pass over the two clips (vt_frame_scores): the
// numbers the reference's evaluation loop publishes (scripts/inference_evaluate.py:175-186 with compute_psnr / compute_ssim,
// vidtok/modules/util.py:146-231), with the script's preprocessing folded into the load:
//   v -> clamp(v, -1, 1) -> (v + 1) / 2, PSNR = -10 log10(mean((x - y)^2) + 1e-8) over C x H x W of a frame,
//   SSIM = mean over channels of the mean of the SSIM map of avg_pool2d(frame, f), f = max(1, round(min(H, W) / 256)),
//   11-tap Gaussian window (sigma 1.5) without padding, c1 = 1e-4, c2 = 9e-4.
// The script clamps only the reconstruction; both clips are clamped here, which is the identity on an input clip that is
// in [-1, 1] as the script's loader makes it.
//
// Arithmetic.  The window moments are taken of u = clamp(v) / 2 = (v + 1) / 2 - 1/2, which is exact in fp32, and the means get
// their 1/2 back afterwards: variances and the covariance do not depend on the shift, x - y does not either, and the
// cancellation in E[u^2] - E[u]^2 loses fewer bits around 0 than around 1/2.  The 2-D window is the product of two normalised
// 1-D windows (equal to the reference's normalised 2-D window in real arithmetic).  x and y go through the same operations
// in the same order, so equal clips give SSIM 1 and PSNR -10 log10(1e-8) exactly.
//
// One CTA takes one tile of kTH x kTW SSIM-map positions of one (batch, channel, frame) plane: it stages the pooled
// (kTH + 10) x (kTW + 10) window of u_x and u_y in shared memory (pooling while loading), runs the row pass over the five
// moments x, y, x^2, y^2, xy into shared memory, the column pass in registers, and writes the tile's (squared-error sum,
// SSIM-map sum) to the workspace.  Every source pixel is counted in the squared error by exactly one tile: a tile owns the
// source pixels under its kTH x kTW pooled pixels, the last tile of a row / column also the window's halo and the rows /
// columns the pooling drops.  A second kernel adds each frame's partials in a fixed order in double.  No atomics anywhere:
// the same input gives the same bits.
#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace vt {

// fp16 beside common.cuh's fp32 / bf16 element helpers (same overload set, so not in the unnamed namespace)
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
__device__ __forceinline__ void load4(const __half* p, float (&o)[4]) {
  uint2 v = *reinterpret_cast<const uint2*>(p);
  const float2 a = __half22float2(*reinterpret_cast<__half2*>(&v.x)), b = __half22float2(*reinterpret_cast<__half2*>(&v.y));
  o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
}

namespace {

constexpr int kThreads = 256;
constexpr int kWin = 11;
constexpr int kTW = 64, kTH = 32;                  // SSIM-map positions per tile
constexpr int kRows = kTH + kWin - 1;              // pooled window rows
constexpr int kCols = kTW + kWin - 1;              // pooled window columns
constexpr int kPitch = (kCols + 3) & ~3;           // the row pass reads whole float4
constexpr int kColThreads = kTW;                   // column pass: one thread per map column and run of kRun rows
constexpr int kRun = kTH / (kThreads / kColThreads);
constexpr size_t kSmem = (size_t)(2 * kRows * kPitch + 5 * kRows * kTW + 2 * (kThreads / 32)) * sizeof(float);
static_assert(kRun * (kThreads / kColThreads) == kTH && kTW % 4 == 0, "tile shape");

// exp(-(i - 5)^2 / (2 * 1.5^2)) / sum, evaluated in double
__device__ constexpr float kG[kWin] = {1.028380084e-03f, 7.598758135e-03f, 3.600077213e-02f, 1.093606895e-01f,
                                       2.130055377e-01f, 2.660117249e-01f, 2.130055377e-01f, 1.093606895e-01f,
                                       3.600077213e-02f, 7.598758135e-03f, 1.028380084e-03f};

// clamp(v, -1, 1) / 2 = (clamp(v) + 1) / 2 - 1/2
__device__ __forceinline__ float half_unit(float v) { return 0.5f * fminf(fmaxf(v, -1.0f), 1.0f); }

struct ScoreGeom {
  int C, T, H, W;
  int f, Hp, Wp;          // pool factor, pooled frame
  int Ho, Wo;             // SSIM map (<= 0: the frame has none)
  int tiles_x, tiles_y;
  int vec;                // rows are read four elements at a time (f in {1, 2, 4}, W % 4 == 0, aligned bases)
  int ssim;
};

// Squared error of the source rectangle [y0, y1) x [x0, x1) of a plane, spread over the CTA
template <typename TX, typename TY>
__device__ __forceinline__ float sse_rect(const TX* __restrict__ xp, const TY* __restrict__ yp, int W, int y0, int y1, int x0, int x1) {
  float s = 0.0f;
  const int w = x1 - x0, n = (y1 - y0) * w;
  for (int it = threadIdx.x; it < n; it += kThreads) {
    const long long o = (long long)(y0 + it / w) * W + x0 + it % w;
    const float d = half_unit(to_f(xp[o])) - half_unit(to_f(yp[o]));
    s = fmaf(d, d, s);
  }
  return s;
}

// Stage the pooled window, four source columns of F source rows per step.  Returns the thread's share of the squared error
// of the owned pixels.  Without the SSIM part only the owned pixels are read.
template <typename TX, typename TY, int F>
__device__ __forceinline__ float stage_vec(const TX* __restrict__ xp, const TY* __restrict__ yp, int W, int sy0, int sx0, int nr, int nc,
                                           int own_h, int own_w, bool all, float* __restrict__ px, float* __restrict__ py) {
  constexpr int P = 4 / F;   // pooled pixels per step
  const int ng = (nc * F + 3) / 4, own_g = own_w * F / 4;
  float sse = 0.0f;
  for (int it = threadIdx.x; it < nr * ng; it += kThreads) {
    const int wy = it / ng, g = it % ng;
    const bool owned = wy < own_h && g < own_g;
    if (!all && !owned) continue;
    float ax[P] = {}, ay[P] = {}, d2 = 0.0f;
#pragma unroll
    for (int r = 0; r < F; ++r) {
      const long long o = (long long)(sy0 + wy * F + r) * W + sx0 + 4 * g;
      float a[4], b[4];
      load4(xp + o, a);
      load4(yp + o, b);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float ua = half_unit(a[j]), ub = half_unit(b[j]), d = ua - ub;
        d2 = fmaf(d, d, d2);
        ax[j / F] += ua;
        ay[j / F] += ub;
      }
    }
    if (owned) sse += d2;
#pragma unroll
    for (int k = 0; k < P; ++k) {
      px[wy * kPitch + g * P + k] = ax[k] * (1.0f / (F * F));
      py[wy * kPitch + g * P + k] = ay[k] * (1.0f / (F * F));
    }
  }
  return sse;
}

// The same for any pool factor and alignment: one pooled pixel per step
template <typename TX, typename TY>
__device__ __forceinline__ float stage_any(const TX* __restrict__ xp, const TY* __restrict__ yp, int W, int f, int sy0, int sx0, int nr,
                                           int nc, int own_h, int own_w, bool all, float* __restrict__ px, float* __restrict__ py) {
  const float area = (float)(f * f);
  float sse = 0.0f;
  for (int it = threadIdx.x; it < nr * nc; it += kThreads) {
    const int wy = it / nc, wx = it % nc;
    const bool owned = wy < own_h && wx < own_w;
    if (!all && !owned) continue;
    float ax = 0.0f, ay = 0.0f, d2 = 0.0f;
    for (int r = 0; r < f; ++r) {
      const long long o = (long long)(sy0 + wy * f + r) * W + sx0 + wx * f;
      for (int j = 0; j < f; ++j) {
        const float ua = half_unit(to_f(xp[o + j])), ub = half_unit(to_f(yp[o + j])), d = ua - ub;
        d2 = fmaf(d, d, d2);
        ax += ua;
        ay += ub;
      }
    }
    if (owned) sse += d2;
    px[wy * kPitch + wx] = __fdiv_rn(ax, area);
    py[wy * kPitch + wx] = __fdiv_rn(ay, area);
  }
  return sse;
}

// Sum over the CTA in a fixed order: butterfly within each warp, then the warps one after the other.  Valid in thread 0.
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.0f;
  if (threadIdx.x == 0)
    for (int w = 0; w < kThreads / 32; ++w) s += red[w];
  return s;
}

template <typename TX, typename TY>
__global__ void __launch_bounds__(kThreads, 2) frame_scores_kernel(const TX* __restrict__ x, const TY* __restrict__ y, ScoreGeom g,
                                                                  float2* __restrict__ part) {
  extern __shared__ __align__(16) float smem[];
  float* px = smem;
  float* py = px + kRows * kPitch;
  float* rp = py + kRows * kPitch;                 // [5][kRows][kTW]
  float* red = rp + 5 * kRows * kTW;

  const int tiles = g.tiles_x * g.tiles_y;
  const long long plane = blockIdx.x / tiles;      // (b * C + c) * T + t
  const int tile = blockIdx.x % tiles;
  const int ty = tile / g.tiles_x, tx = tile % g.tiles_x;
  const bool last_y = ty == g.tiles_y - 1, last_x = tx == g.tiles_x - 1;
  const int oy0 = ty * kTH, ox0 = tx * kTW;
  const int nr = min(kRows, g.Hp - oy0), nc = min(kCols, g.Wp - ox0);      // staged pooled window
  const int own_h = last_y ? nr : kTH, own_w = last_x ? nc : kTW;
  const TX* xp = x + plane * g.H * g.W;
  const TY* yp = y + plane * g.H * g.W;
  const int f = g.f, sy0 = oy0 * f, sx0 = ox0 * f;

  float sse;
  if (g.vec && f == 1) sse = stage_vec<TX, TY, 1>(xp, yp, g.W, sy0, sx0, nr, nc, own_h, own_w, g.ssim, px, py);
  else if (g.vec && f == 2) sse = stage_vec<TX, TY, 2>(xp, yp, g.W, sy0, sx0, nr, nc, own_h, own_w, g.ssim, px, py);
  else if (g.vec) sse = stage_vec<TX, TY, 4>(xp, yp, g.W, sy0, sx0, nr, nc, own_h, own_w, g.ssim, px, py);
  else sse = stage_any(xp, yp, g.W, f, sy0, sx0, nr, nc, own_h, own_w, g.ssim, px, py);
  // the columns and rows the pooling drops belong to the last tiles
  if (last_x && g.Wp * f < g.W) sse += sse_rect(xp, yp, g.W, sy0, last_y ? g.H : sy0 + kTH * f, g.Wp * f, g.W);
  if (last_y && g.Hp * f < g.H) sse += sse_rect(xp, yp, g.W, g.Hp * f, g.H, sx0, last_x ? g.Wp * f : sx0 + kTW * f);
  __syncthreads();

  float ssum = 0.0f;
  if (g.ssim) {
    const int now = min(kTW, g.Wo - ox0), noh = min(kTH, g.Ho - oy0);      // map positions of this tile
    // row pass: four neighbouring outputs of the five moments from sixteen staged values
    for (int it = threadIdx.x; it < nr * (kTW / 4); it += kThreads) {
      const int wy = it / (kTW / 4), q = it % (kTW / 4);
      if (4 * q >= now) continue;
      float a[16], b[16];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float4 va = *reinterpret_cast<const float4*>(px + wy * kPitch + 4 * q + 4 * k);
        const float4 vb = *reinterpret_cast<const float4*>(py + wy * kPitch + 4 * q + 4 * k);
        a[4 * k] = va.x; a[4 * k + 1] = va.y; a[4 * k + 2] = va.z; a[4 * k + 3] = va.w;
        b[4 * k] = vb.x; b[4 * k + 1] = vb.y; b[4 * k + 2] = vb.z; b[4 * k + 3] = vb.w;
      }
      float acc[5][4] = {};
#pragma unroll
      for (int k = 0; k < kWin + 3; ++k) {
        const float m[5] = {a[k], b[k], __fmul_rn(a[k], a[k]), __fmul_rn(b[k], b[k]), __fmul_rn(a[k], b[k])};
#pragma unroll
        for (int o = 0; o < 4; ++o)
          if (k - o >= 0 && k - o < kWin)
#pragma unroll
            for (int c = 0; c < 5; ++c) acc[c][o] = __fmaf_rn(kG[k - o], m[c], acc[c][o]);
      }
#pragma unroll
      for (int c = 0; c < 5; ++c)
        *reinterpret_cast<float4*>(rp + (c * kRows + wy) * kTW + 4 * q) = make_float4(acc[c][0], acc[c][1], acc[c][2], acc[c][3]);
    }
    __syncthreads();

    // column pass: kRun outputs of one map column slide over kRun + 10 rows of the row pass
    const int ox = threadIdx.x % kColThreads, r0 = (threadIdx.x / kColThreads) * kRun;
    if (ox < now && r0 < noh) {
      float acc[5][kRun] = {};
#pragma unroll
      for (int i = 0; i < kRun + kWin - 1; ++i) {
        float m[5];
#pragma unroll
        for (int c = 0; c < 5; ++c) m[c] = rp[(c * kRows + r0 + i) * kTW + ox];
#pragma unroll
        for (int r = 0; r < kRun; ++r)
          if (i - r >= 0 && i - r < kWin)
#pragma unroll
            for (int c = 0; c < 5; ++c) acc[c][r] = __fmaf_rn(kG[i - r], m[c], acc[c][r]);
      }
      constexpr float c1 = 1e-4f, c2 = 9e-4f;   // (0.01 * data_range)^2, (0.03 * data_range)^2
#pragma unroll
      for (int r = 0; r < kRun; ++r) {
        const float ux = acc[0][r], uy = acc[1][r];
        const float sxx = __fsub_rn(acc[2][r], __fmul_rn(ux, ux)), syy = __fsub_rn(acc[3][r], __fmul_rn(uy, uy));
        const float sxy = __fsub_rn(acc[4][r], __fmul_rn(ux, uy));
        const float mx = __fadd_rn(ux, 0.5f), my = __fadd_rn(uy, 0.5f);
        const float mxx = __fmul_rn(mx, mx), myy = __fmul_rn(my, my), mxy = __fmul_rn(mx, my);
        const float cs = __fdiv_rn(__fadd_rn(__fadd_rn(sxy, sxy), c2), __fadd_rn(__fadd_rn(sxx, syy), c2));
        const float lum = __fdiv_rn(__fadd_rn(__fadd_rn(mxy, mxy), c1), __fadd_rn(__fadd_rn(mxx, myy), c1));
        if (r0 + r < noh) ssum += __fmul_rn(lum, cs);
      }
    }
  }

  const float tile_sse = block_sum(sse, red);
  __syncthreads();
  const float tile_ssim = block_sum(ssum, red);
  if (threadIdx.x == 0) {
    const long long frame = (plane / ((long long)g.C * g.T)) * g.T + plane % g.T;
    const int c = (int)((plane / g.T) % g.C);
    part[(frame * g.C + c) * tiles + tile] = make_float2(tile_sse, tile_ssim);
  }
}

// Per frame: the partials of its C * tiles tiles added in index order in double, then the two scores.  Thread 0 then adds the
// call's frames, in frame order, to the caller's running [sum of PSNR, sum of SSIM, frames].
__global__ void __launch_bounds__(kThreads) frame_scores_finish_kernel(const float2* __restrict__ part, long long frames, int per_frame,
                                                                      double n_px, double n_map, float* __restrict__ psnr,
                                                                      float* __restrict__ ssim, double* __restrict__ running) {
  for (long long fr = threadIdx.x; fr < frames; fr += kThreads) {
    double e = 0.0, s = 0.0;
    for (int i = 0; i < per_frame; ++i) {
      const float2 v = part[fr * per_frame + i];
      e += (double)v.x;
      s += (double)v.y;
    }
    psnr[fr] = (float)(-10.0 * log10(e / n_px + 1e-8));
    if (ssim) ssim[fr] = (float)(s / n_map);
  }
  __syncthreads();
  if (running && threadIdx.x == 0) {
    double p = running[0], s = running[1];
    for (long long fr = 0; fr < frames; ++fr) {
      p += (double)psnr[fr];
      if (ssim) s += (double)ssim[fr];
    }
    running[0] = p;
    running[1] = s;
    running[2] += (double)frames;
  }
}

bool make_geom(int B, int C, int T, int H, int W, ScoreGeom& g) {
  g.C = C; g.T = T; g.H = H; g.W = W;
  g.f = frame_scores_pool_factor(H, W);
  g.Hp = H / g.f; g.Wp = W / g.f;
  g.Ho = g.Hp - (kWin - 1); g.Wo = g.Wp - (kWin - 1);
  g.tiles_x = std::max(1, (g.Wo + kTW - 1) / kTW);
  g.tiles_y = std::max(1, (g.Ho + kTH - 1) / kTH);
  g.vec = 0;
  g.ssim = 0;
  return (long long)B * C * T * g.tiles_x * g.tiles_y <= 0x7fffffffLL;
}

template <typename TX, typename TY>
cudaError_t launch_typed(const void* x, const void* y, ScoreGeom g, long long planes, float2* part, cudaStream_t s) {
  g.vec = (g.f == 1 || g.f == 2 || g.f == 4) && g.W % 4 == 0 && (uintptr_t)x % (4 * sizeof(TX)) == 0 && (uintptr_t)y % (4 * sizeof(TY)) == 0;
  cudaError_t e = cudaFuncSetAttribute(frame_scores_kernel<TX, TY>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem);
  if (e != cudaSuccess) return e;
  frame_scores_kernel<TX, TY><<<(unsigned)(planes * g.tiles_x * g.tiles_y), kThreads, kSmem, s>>>((const TX*)x, (const TY*)y, g, part);
  return cudaGetLastError();
}

template <typename TX>
cudaError_t launch_x_typed(const void* x, const void* y, int y_dtype, const ScoreGeom& g, long long planes, float2* part, cudaStream_t s) {
  switch (y_dtype) {
    case 0: return launch_typed<TX, float>(x, y, g, planes, part, s);
    case 1: return launch_typed<TX, bf16>(x, y, g, planes, part, s);
    case 2: return launch_typed<TX, __half>(x, y, g, planes, part, s);
  }
  return cudaErrorInvalidValue;
}

}  // namespace

// max(1, round(min(H, W) / 256)) with Python's round (half to even)
int frame_scores_pool_factor(int H, int W) {
  const int m = std::min(H, W), q = m / 256, r = m % 256;
  const int rounded = r > 128 ? q + 1 : (r < 128 ? q : q + (q & 1));
  return std::max(1, rounded);
}

bool frame_scores_has_ssim(int H, int W) {
  const int f = frame_scores_pool_factor(H, W);
  return H / f >= kWin && W / f >= kWin;
}

long long frame_scores_workspace(int B, int C, int T, int H, int W) {
  ScoreGeom g;
  if (!make_geom(B, C, T, H, W, g)) return -1;
  return (long long)B * C * T * g.tiles_x * g.tiles_y * (long long)sizeof(float2);
}

cudaError_t launch_frame_scores(const void* x, int x_dtype, const void* y, int y_dtype, int B, int C, int T, int H, int W, float* psnr,
                                float* ssim, double* running, void* ws, cudaStream_t s) {
  ScoreGeom g;
  if (!make_geom(B, C, T, H, W, g) || (ssim && (g.Ho <= 0 || g.Wo <= 0))) return cudaErrorInvalidValue;
  g.ssim = ssim != nullptr;
  const long long planes = (long long)B * C * T, frames = (long long)B * T, elems = planes * H * W;
  float2* part = static_cast<float2*>(ws);
  {
    // algorithmic bytes: both clips read once
    ProfScope _ps("frame_scores", 0.0, (double)elems * (double)((x_dtype == 0 ? 4 : 2) + (y_dtype == 0 ? 4 : 2)), s);
    cudaError_t e = cudaErrorInvalidValue;
    switch (x_dtype) {
      case 0: e = launch_x_typed<float>(x, y, y_dtype, g, planes, part, s); break;
      case 1: e = launch_x_typed<bf16>(x, y, y_dtype, g, planes, part, s); break;
      case 2: e = launch_x_typed<__half>(x, y, y_dtype, g, planes, part, s); break;
    }
    if (e != cudaSuccess) return e;
    count_launch();
  }
  const int per_frame = C * g.tiles_x * g.tiles_y;
  ProfScope _ps("frame_scores_finish", 0.0, (double)frames * (per_frame * 8.0 + 8.0), s);
  frame_scores_finish_kernel<<<1, kThreads, 0, s>>>(part, frames, per_frame, (double)C * H * W, (double)C * g.Ho * g.Wo, psnr, ssim, running);
  count_launch();
  return cudaGetLastError();
}

}  // namespace vt
