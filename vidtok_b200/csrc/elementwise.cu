// Bandwidth-bound kernels of the path: per-position LayerNorm(+SiLU), GroupNorm(+SiLU), softmax rows,
// KL reparameterisation, FSQ quantiser, weight repacking, trilinear time interpolation.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace vt {

thread_local long long g_launches = 0;

thread_local bool g_prof_on = false;
static bool g_prof_on_flag() { return g_prof_on; }
struct ProfRec { std::string name; double flops, bytes; cudaEvent_t e0, e1; };
thread_local bool g_prof_detail = false;
bool prof_enabled() { return g_prof_on_flag(); }

thread_local std::vector<ProfRec> g_prof;
thread_local std::vector<cudaEvent_t> g_prof_pool;
static cudaEvent_t prof_event() {
  cudaEvent_t e;
  if (!g_prof_pool.empty()) { e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
  cudaEventCreate(&e);
  return e;
}
ProfScope::ProfScope(const char* name, double flops, double bytes, cudaStream_t stream, const char* detail) : idx(-1), s(stream) {
  if (!g_prof_on) return;
  std::string nm = name;
  if (g_prof_detail && detail) { nm += " "; nm += detail; }
  ProfRec r{nm, flops, bytes, prof_event(), prof_event()};
  cudaEventRecord(r.e0, s);
  idx = (int)g_prof.size();
  g_prof.push_back(r);
}
ProfScope::~ProfScope() {
  if (idx >= 0) cudaEventRecord(g_prof[idx].e1, s);
}
void prof_set_detail(bool on) { g_prof_detail = on; }
void prof_start() {
  for (auto& r : g_prof) { g_prof_pool.push_back(r.e0); g_prof_pool.push_back(r.e1); }
  g_prof.clear();
  g_prof_on = true;
}
// aggregates per kernel name into a JSON object; returns the number of bytes written (0 if it does not fit)
int prof_stop(char* buf, int cap) {
  g_prof_on = false;
  // wait for the profiled kernels' own events rather than the device: a device-wide synchronise would break a CUDA graph
  // that another stream is capturing (the tokenizer refuses to launch under capture while the profiler is on)
  for (auto& r : g_prof) cudaEventSynchronize(r.e1);
  struct Agg { std::string name; long long n; double ms, flops, bytes; };
  std::vector<Agg> aggs;
  for (auto& r : g_prof) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, r.e0, r.e1);
    Agg* a = nullptr;
    for (auto& x : aggs) if (x.name == r.name) a = &x;
    if (!a) { aggs.push_back({r.name, 0, 0, 0, 0}); a = &aggs.back(); }
    a->n++; a->ms += ms; a->flops += r.flops; a->bytes += r.bytes;
    g_prof_pool.push_back(r.e0); g_prof_pool.push_back(r.e1);
  }
  g_prof.clear();
  std::string out = "{";
  for (size_t i = 0; i < aggs.size(); ++i) {
    char tmp[512];
    snprintf(tmp, sizeof(tmp), "%s\"%s\": {\"launches\": %lld, \"ms\": %.6f, \"flops\": %.6e, \"bytes\": %.6e}", i ? ", " : "",
             aggs[i].name.c_str(), aggs[i].n, aggs[i].ms, aggs[i].flops, aggs[i].bytes);
    out += tmp;
  }
  out += "}";
  if ((int)out.size() + 1 > cap) return 0;
  memcpy(buf, out.c_str(), out.size() + 1);
  return (int)out.size();
}

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
template <bool EXACT> __device__ __forceinline__ float act_silu(float x) {
  return EXACT ? silu_exact(x) : silu_f(x);
}

// ---- row accessors: one code path for plain (fp32 / bf16) rows and hi|lo split rows (DT_SPLIT, kernels.h) ----------
// A split row of C logical channels is 2*C bf16 values: [hi(C) | lo(C)], value = hi + lo.
struct split16 { bf16 v; };
template <typename T> struct RowAcc {
  static constexpr int W = 1;
  static __device__ __forceinline__ float ld(const T* row, int C, int c) { return to_f(row[c]); }
  static __device__ __forceinline__ void st(T* row, int C, int c, float v) { row[c] = from_f<T>(v); }
};
template <> struct RowAcc<split16> {
  static constexpr int W = 2;
  static __device__ __forceinline__ float ld(const split16* row, int C, int c) { return split_load(&row[c].v, &row[C + c].v); }
  static __device__ __forceinline__ void st(split16* row, int C, int c, float v) { split_store(&row[c].v, &row[C + c].v, v); }
};
__device__ __forceinline__ void split8(const float (&f)[8], uint4& hi, uint4& lo) {
  __half2* h2 = reinterpret_cast<__half2*>(&hi);
  __half2* l2 = reinterpret_cast<__half2*>(&lo);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    h2[i] = __floats2half2_rn(split_sat(f[2 * i]), split_sat(f[2 * i + 1]));
    const float2 hf = __half22float2(h2[i]);
    l2[i] = __floats2half2_rn(split_sat(f[2 * i] - hf.x), split_sat(f[2 * i + 1] - hf.y));
  }
}
__device__ __forceinline__ void join8(const uint4& hi, const uint4& lo, float (&f)[8]) {
  const __half2* h2 = reinterpret_cast<const __half2*>(&hi);
  const __half2* l2 = reinterpret_cast<const __half2*>(&lo);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 a = __half22float2(h2[i]), b = __half22float2(l2[i]);
    f[2 * i] = a.x + b.x;
    f[2 * i + 1] = a.y + b.y;
  }
}
// LayerNorm(+SiLU) of split rows (EXACT_TC mode, C % 8 == 0): one warp per position, fp32 two-pass statistics.  Rows of up
// to 512 channels (every LayerNorm of the model zoo) stay in registers: one read of x, one write of y; longer rows re-read
// x from L1 for the second and third pass.
template <bool SILU>
__global__ void __launch_bounds__(256) layernorm_split_kernel(const bf16* __restrict__ x, const float* __restrict__ gamma,
                                                              const float* __restrict__ beta, bf16* __restrict__ y,
                                                              long long rows, int C) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const bf16* xr = x + row * 2 * C;
  bf16* yr = y + row * 2 * C;
  if (C <= 512) {
    float f[2][8];
    const int c0 = lane * 8, c1 = lane * 8 + 256;
    const bool h0 = c0 < C, h1 = c1 < C;
#pragma unroll
    for (int i = 0; i < 8; ++i) f[0][i] = f[1][i] = 0.f;
    if (h0) join8(__ldg(reinterpret_cast<const uint4*>(xr + c0)), __ldg(reinterpret_cast<const uint4*>(xr + C + c0)), f[0]);
    if (h1) join8(__ldg(reinterpret_cast<const uint4*>(xr + c1)), __ldg(reinterpret_cast<const uint4*>(xr + C + c1)), f[1]);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += f[0][i];
#pragma unroll
    for (int i = 0; i < 8; ++i) s += f[1][i];
    const float mean = warp_sum(s) / (float)C;
    float q = 0.f;
    if (h0) {
#pragma unroll
      for (int i = 0; i < 8; ++i) { const float d = f[0][i] - mean; q = fmaf(d, d, q); }
    }
    if (h1) {
#pragma unroll
      for (int i = 0; i < 8; ++i) { const float d = f[1][i] - mean; q = fmaf(d, d, q); }
    }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)C + 1e-6f);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int c = k ? c1 : c0;
      if (!(k ? h1 : h0)) continue;
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c + 4));
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c + 4));
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float t = (f[k][i] - mean) * rstd * gg[i] + bb[i];
        f[k][i] = SILU ? silu_tc(t) : t;
      }
      uint4 hi, lo;
      split8(f[k], hi, lo);
      *reinterpret_cast<uint4*>(yr + c) = hi;
      *reinterpret_cast<uint4*>(yr + C + c) = lo;
    }
    return;
  }
  float s = 0.f;
  for (int c = lane * 8; c < C; c += 256) {
    float f[8];
    join8(*reinterpret_cast<const uint4*>(xr + c), *reinterpret_cast<const uint4*>(xr + C + c), f);
#pragma unroll
    for (int i = 0; i < 8; ++i) s += f[i];
  }
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
  for (int c = lane * 8; c < C; c += 256) {
    float f[8];
    join8(*reinterpret_cast<const uint4*>(xr + c), *reinterpret_cast<const uint4*>(xr + C + c), f);
#pragma unroll
    for (int i = 0; i < 8; ++i) { const float d = f[i] - mean; q = fmaf(d, d, q); }
  }
  const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)C + 1e-6f);
  for (int c = lane * 8; c < C; c += 256) {
    float f[8];
    join8(*reinterpret_cast<const uint4*>(xr + c), *reinterpret_cast<const uint4*>(xr + C + c), f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float t = (f[i] - mean) * rstd * gamma[c + i] + beta[c + i];
      f[i] = SILU ? silu_tc(t) : t;
    }
    uint4 hi, lo;
    split8(f, hi, lo);
    *reinterpret_cast<uint4*>(yr + c) = hi;
    *reinterpret_cast<uint4*>(yr + C + c) = lo;
  }
}

// ---- LayerNorm over channels (model_3dcausal.py:62-80; eps 1e-6, affine), optional SiLU (:26-27) --------
// One warp per position; VPL vectors of 4 channels per lane held in registers (C == 128*VPL).
template <typename T, int VPL, bool SILU, bool EXACT>
__global__ void __launch_bounds__(256) layernorm_vec_kernel(const T* __restrict__ x, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, T* __restrict__ y,
                                                            long long rows) {
  constexpr int C = 128 * VPL;
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const T* xr = x + row * C;
  float v[VPL][4];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    load4(xr + (i * 32 + lane) * 4, v[i]);
    s += (v[i][0] + v[i][1]) + (v[i][2] + v[i][3]);
  }
  const float mean = warp_sum(s) * (1.0f / C);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float d = v[i][j] - mean;
      q = fmaf(d, d, q);
    }
  const float var = warp_sum(q) * (1.0f / C);
  const float rstd = EXACT ? (1.0f / sqrtf(var + 1e-6f)) : rsqrtf(var + 1e-6f);
  T* yr = y + row * C;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c = (i * 32 + lane) * 4;
    float g[4], b[4], o[4];
    load4(gamma + c, g);
    load4(beta + c, b);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float t = (v[i][j] - mean) * rstd * g[j] + b[j];
      o[j] = SILU ? act_silu<EXACT>(t) : t;
    }
    store4(yr + c, o);
  }
}

// bf16 fast path: persistent warps, 16-byte loads (8 channels per lane), two row-groups in flight per warp.
// C = 128: half a warp per row (two rows per warp pass); C = 256: one warp per row; C = 512: two vectors per lane.
template <int C, bool SILU>
__global__ void __launch_bounds__(256) layernorm_bf16_kernel(const bf16* __restrict__ x, const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, bf16* __restrict__ y,
                                                             long long rows) {
  constexpr int LPR = (C / 8) < 32 ? (C / 8) : 32;  // lanes per row
  constexpr int V = C / (8 * LPR);                  // 16-byte vectors per lane
  constexpr int RPW = 32 / LPR;                     // rows per warp pass
  constexpr int U = (V == 1) ? 4 : 2;               // passes in flight (64 B per lane outstanding)
  const int lane = threadIdx.x & 31, sub = lane / LPR, l = lane % LPR;
  const long long gw = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * 8;
  float g[V][8], b[V][8];
#pragma unroll
  for (int v = 0; v < V; ++v) {
    const int c = (v * LPR + l) * 8;
    float4 t0 = *reinterpret_cast<const float4*>(gamma + c), t1 = *reinterpret_cast<const float4*>(gamma + c + 4);
    g[v][0] = t0.x; g[v][1] = t0.y; g[v][2] = t0.z; g[v][3] = t0.w; g[v][4] = t1.x; g[v][5] = t1.y; g[v][6] = t1.z; g[v][7] = t1.w;
    t0 = *reinterpret_cast<const float4*>(beta + c); t1 = *reinterpret_cast<const float4*>(beta + c + 4);
    b[v][0] = t0.x; b[v][1] = t0.y; b[v][2] = t0.z; b[v][3] = t0.w; b[v][4] = t1.x; b[v][5] = t1.y; b[v][6] = t1.z; b[v][7] = t1.w;
  }
  for (long long r0 = gw * (RPW * U); r0 < rows; r0 += nw * (RPW * U)) {
    uint4 raw[U][V];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long row = r0 + u * RPW + sub;
#pragma unroll
      for (int v = 0; v < V; ++v)
        raw[u][v] = row < rows ? *reinterpret_cast<const uint4*>(x + row * C + (v * LPR + l) * 8) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long row = r0 + u * RPW + sub;
      float f[V][8];
      float s = 0.f;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw[u][v]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          f[v][2 * i] = __low2float(h[i]);
          f[v][2 * i + 1] = __high2float(h[i]);
          s += f[v][2 * i] + f[v][2 * i + 1];
        }
      }
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float mean = s * (1.0f / C);
      float q = 0.f;
#pragma unroll
      for (int v = 0; v < V; ++v)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = f[v][i] - mean;
          q = fmaf(d, d, q);
        }
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      const float rstd = rsqrtf(q * (1.0f / C) + 1e-6f);
      const float nmr = -mean * rstd;
      if (row < rows) {
#pragma unroll
        for (int v = 0; v < V; ++v) {
          uint4 o4;
          __nv_bfloat162* ho = reinterpret_cast<__nv_bfloat162*>(&o4);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            // ((x - mean) * rstd) * g + b with xhat = fma(x, rstd, -mean*rstd)
            float a0 = fmaf(fmaf(f[v][2 * i], rstd, nmr), g[v][2 * i], b[v][2 * i]);
            float a1 = fmaf(fmaf(f[v][2 * i + 1], rstd, nmr), g[v][2 * i + 1], b[v][2 * i + 1]);
            if (SILU) { a0 = silu_f(a0); a1 = silu_f(a1); }
            ho[i] = __floats2bfloat162_rn(a0, a1);
          }
          *reinterpret_cast<uint4*>(y + row * C + (v * LPR + l) * 8) = o4;
        }
      }
    }
  }
}

// generic C (tiny test models): one warp per position, strided scalar access
template <typename T, bool SILU, bool EXACT>
__global__ void __launch_bounds__(256) layernorm_gen_kernel(const T* __restrict__ x, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, T* __restrict__ y,
                                                            long long rows, int C) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  using A = RowAcc<T>;
  const T* xr = x + row * C * A::W;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += A::ld(xr, C, c);
  const float mean = warp_sum(s) / C;
  float q = 0.f;
  for (int c = lane; c < C; c += 32) {
    float d = A::ld(xr, C, c) - mean;
    q = fmaf(d, d, q);
  }
  const float var = warp_sum(q) / C;
  const float rstd = 1.0f / sqrtf(var + 1e-6f);
  T* yr = y + row * C * A::W;
  for (int c = lane; c < C; c += 32) {
    float t = (A::ld(xr, C, c) - mean) * rstd * gamma[c] + beta[c];
    A::st(yr, C, c, SILU ? act_silu<EXACT>(t) : t);
  }
}

// ---- GroupNorm(32 groups, eps 1e-6) per frame (model_3dcausal.py:30-32 applied on `(b t) c h w`) -----------
// stats pass: one block per (frame, group): two-pass mean / variance over (positions x C/32)
template <typename T>
__global__ void __launch_bounds__(256) groupnorm_stats_kernel(const T* __restrict__ x, float* __restrict__ stats,
                                                              long long pos_per_frame, int C) {
  const int cpg = C / 32;
  const long long frame = blockIdx.x / 32;
  const int g = blockIdx.x % 32;
  using A = RowAcc<T>;
  const T* base = x + frame * pos_per_frame * C * A::W;
  const long long n = pos_per_frame * cpg;
  __shared__ float red[32];
  __shared__ float bc;
  auto block_sum = [&](float v) -> float {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
      float t = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
      t = warp_sum(t);
      if (threadIdx.x == 0) bc = t;
    }
    __syncthreads();
    float r = bc;
    __syncthreads();
    return r;
  };
  float s = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) s += A::ld(base + (i / cpg) * C * A::W, C, g * cpg + (int)(i % cpg));
  const float mean = block_sum(s) / (float)n;
  float q = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    float d = A::ld(base + (i / cpg) * C * A::W, C, g * cpg + (int)(i % cpg)) - mean;
    q = fmaf(d, d, q);
  }
  const float var = block_sum(q) / (float)n;
  if (threadIdx.x == 0) {
    stats[2 * blockIdx.x] = mean;
    stats[2 * blockIdx.x + 1] = 1.0f / sqrtf(var + 1e-6f);
  }
}
template <typename T, bool SILU, bool EXACT>
__global__ void __launch_bounds__(256) groupnorm_apply_kernel(const T* __restrict__ x, const float* __restrict__ stats,
                                                              const float* __restrict__ gamma,
                                                              const float* __restrict__ beta, T* __restrict__ y,
                                                              long long total, long long pos_per_frame, int C) {
  const int cpg = C / 32;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    using A = RowAcc<T>;
    const int c = (int)(i % C);
    const long long pos = i / C;
    const long long frame = pos / pos_per_frame;
    const float* st = stats + 2 * (frame * 32 + c / cpg);
    float t = (A::ld(x + pos * C * A::W, C, c) - st[0]) * st[1] * gamma[c] + beta[c];
    A::st(y + pos * C * A::W, C, c, SILU ? act_silu<EXACT>(t) : t);
  }
}
// per-position variant: statistics over the C/32 channels of one position (the temporal 1D blocks,
// model_3dcausal.py:474-480 -- see oracle/vidtok_oracle.py:norm)
template <typename T, bool SILU, bool EXACT>
__global__ void __launch_bounds__(256) groupnorm_pos_kernel(const T* __restrict__ x, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, T* __restrict__ y,
                                                            long long npos, int C) {
  const int cpg = C / 32;
  const long long total = npos * 32;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long pos = i / 32;
    const int g = (int)(i % 32);
    using A = RowAcc<T>;
    const T* xr = x + pos * C * A::W;
    const int c0 = g * cpg;
    float s = 0.f;
    for (int c = 0; c < cpg; ++c) s += A::ld(xr, C, c0 + c);
    const float mean = s / cpg;
    float q = 0.f;
    for (int c = 0; c < cpg; ++c) {
      float d = A::ld(xr, C, c0 + c) - mean;
      q = fmaf(d, d, q);
    }
    const float rstd = 1.0f / sqrtf(q / cpg + 1e-6f);
    T* yr = y + pos * C * A::W;
    for (int c = 0; c < cpg; ++c) {
      float t = (A::ld(xr, C, c0 + c) - mean) * rstd * gamma[c0 + c] + beta[c0 + c];
      A::st(yr, C, c0 + c, SILU ? act_silu<EXACT>(t) : t);
    }
  }
}

// ---- softmax over rows of fp32 scores -> P (attention, model_3dcausal.py:140) -----------------------------
template <typename TOut>
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ S, TOut* __restrict__ P, int N) {
  using A = RowAcc<TOut>;
  const float* s = S + (long long)blockIdx.x * N;
  TOut* p = P + (long long)blockIdx.x * N * A::W;
  __shared__ float red[8];
  __shared__ float bc;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < N; i += 256) m = fmaxf(m, s[i]);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < 8 ? red[threadIdx.x] : -INFINITY;
    t = warp_max(t);
    if (threadIdx.x == 0) bc = t;
  }
  __syncthreads();
  m = bc;
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x; i < N; i += 256) sum += expf(s[i] - m);
  sum = warp_sum(sum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < 8 ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) bc = t;
  }
  __syncthreads();
  const float inv = 1.0f / bc;
  for (int i = threadIdx.x; i < N; i += 256) A::st(p, N, i, expf(s[i] - m) * inv);
}

// ---- KL: DiagonalGaussianDistribution (distributions.py:5-28) + regularizer (regularizers.py:82-92) ------
// h [B,2z,P] fp32 (NCDHW flattened), noise/z [B,z,P]
__global__ void __launch_bounds__(256) kl_kernel(const float* __restrict__ h, const float* __restrict__ noise, int zc,
                                                 long long P, int B, int sample, float* __restrict__ z,
                                                 double* __restrict__ kl_acc) {
  const long long total = (long long)B * zc * P;
  double local = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / (zc * P), r = i % (zc * P);
    float zv;
    local += (double)kl_sample_one(h[b * 2 * zc * P + r], h[b * 2 * zc * P + zc * P + r], sample ? noise[i] : 0.f, sample, zv);
    z[i] = zv;
  }
  __shared__ double red[8];
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += red[i];
    atomicAdd(kl_acc, t);
  }
}
__global__ void kl_finish_kernel(const double* acc, int B, float* out) { *out = (float)(0.5 * acc[0] / B); }

// ---- FSQ: bound -> round -> index (regularizers.py:153-178,206-262) --------------------------------------
__global__ void __launch_bounds__(256) fsq_kernel(const float* __restrict__ h, FsqConst c, long long P, int B,
                                                  float* __restrict__ codes, int* __restrict__ indices) {
  const long long total = (long long)B * P;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / P, pos = i % P;
    float idx = 0.f;
    for (int k = 0; k < c.d; ++k) {
      codes[(b * c.d + k) * P + pos] = fsq_code(c, k, h[(b * c.d + k) * P + pos], idx);
    }
    if (indices) indices[i] = (int)idx;
  }
}
__global__ void __launch_bounds__(256) fsq_i2c_kernel(const int* __restrict__ indices, FsqConst c, long long P, int B,
                                                      float* __restrict__ codes) {
  const long long total = (long long)B * P;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / P, pos = i % P;
    const int idx = indices[i];
    for (int k = 0; k < c.d; ++k) {
      const int dgt = (idx / c.basis[k]) % c.levels[k];
      const int hw = c.levels[k] / 2;
      codes[(b * c.d + k) * P + pos] = (float)(dgt - hw) / (float)hw;
    }
  }
}
// ---- weight repacking -------------------------------------------------------------------------------------
__global__ void pack_w_kn_kernel(const float* __restrict__ w, float* __restrict__ out, int Co, int Ci, int taps) {
  const long long total = (long long)Co * Ci * taps;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i % Co);
    const long long k = i / Co;
    const int tap = (int)(k / Ci), ci = (int)(k % Ci);
    out[i] = w[((long long)co * Ci + ci) * taps + tap];
  }
}
struct CollapseMap { int mt[3], mh[3], mw[3]; };
// wscale != 0: split rows [hi(K) | lo(K)] (row length 2*K) of fp16 planes of v * wscale (a power of two chosen by the caller
// so that the lo plane stays in fp16's normal range; the conv epilogue undoes it on the accumulator); wscale == 0: bf16 rows
__device__ __forceinline__ void put_w(bf16* out, long long row, int K, int k, float v, float wscale) {
  if (wscale != 0.f) split_store(&out[row * 2 * K + k], &out[row * 2 * K + K + k], v * wscale);
  else out[row * K + k] = __float2bfloat16_rn(v);
}
// max |w| of a tensor (one block; result in *out)
__global__ void __launch_bounds__(1024) absmax_kernel(const float* __restrict__ w, long long n, float* __restrict__ out) {
  float m = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(w[i]));
  m = warp_max(m);
  __shared__ float red[32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_max(t);
    if (threadIdx.x == 0) *out = t;
  }
}
__global__ void pack_w_collapsed_kernel(const float* __restrict__ w, bf16* __restrict__ out, int Co, int Co_pad, int Ci,
                                        int kt, int kh, int kw, CollapseMap cm, int kt2, int kh2, int kw2, float wscale) {
  const int K2 = kt2 * kh2 * kw2 * Ci;
  const long long total = (long long)Co_pad * K2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % K2);
    const int co = (int)(i / K2);
    const int ci = k % Ci, tap2 = k / Ci;
    const int c2 = tap2 % kw2, b2 = (tap2 / kw2) % kh2, a2 = tap2 / (kw2 * kh2);
    float v = 0.f;
    if (co < Co)
      for (int a = 0; a < kt; ++a)
        for (int b = 0; b < kh; ++b)
          for (int c = 0; c < kw; ++c)
            if (cm.mt[a] == a2 && cm.mh[b] == b2 && cm.mw[c] == c2)
              v += w[((long long)co * Ci + ci) * (kt * kh * kw) + (a * kh + b) * kw + c];
    put_w(out, co, K2, k, v, wscale);
  }
}
__global__ void pack_w_nk_bf16_kernel(const float* __restrict__ w, bf16* __restrict__ out, int Co, int Co_pad, int Ci, int taps,
                                      int Kpad, float wscale) {
  const long long total = (long long)Co_pad * Kpad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % Kpad);
    const int co = (int)(i / Kpad);
    float v = 0.f;
    if (co < Co && k < Ci * taps) {
      const int tap = k / Ci, ci = k % Ci;
      v = w[((long long)co * Ci + ci) * taps + tap];
    }
    put_w(out, co, Kpad, k, v, wscale);
  }
}

// ---- trilinear 2x along T (F.interpolate(scale_factor=[2,1,1], mode="trilinear"), model_3dcausal_v1_1.py:328-339)
template <typename T>
__global__ void __launch_bounds__(256) time_interp2x_kernel(const T* __restrict__ x, T* __restrict__ y, int B, int Tn,
                                                            long long hwc) {
  // 4 elements per thread (hwc is a multiple of 4: channels-last with C % 4 == 0)
  const long long q = hwc / 4;
  const long long total = (long long)B * 2 * Tn * q;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long e = (i % q) * 4;
    const long long r = i / q;
    const int j = (int)(r % (2 * Tn));
    const long long b = r / (2 * Tn);
    float src = 0.5f * ((float)j + 0.5f) - 0.5f;
    src = src < 0.f ? 0.f : src;
    const int i0 = (int)src;
    const int i1 = i0 + ((i0 < Tn - 1) ? 1 : 0);
    const float l1 = src - (float)i0, l0 = 1.0f - l1;
    float a[4], c[4], o[4];
    load4(x + (b * Tn + i0) * hwc + e, a);
    load4(x + (b * Tn + i1) * hwc + e, c);
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = __fadd_rn(__fmul_rn(l0, a[k]), __fmul_rn(l1, c[k]));
    store4(y + (b * 2 * Tn + j) * hwc + e, o);
  }
}
// bf16, 8 elements (16 bytes) per thread, same arithmetic
__global__ void __launch_bounds__(256) time_interp2x_bf16x8_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int B, int Tn,
                                                                   long long hwc) {
  const long long q = hwc / 8;
  const long long total = (long long)B * 2 * Tn * q;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / q;
    const long long e = (i - r * q) * 8;
    const int j = (int)(r % (2 * Tn));
    const long long b = r / (2 * Tn);
    float src = 0.5f * ((float)j + 0.5f) - 0.5f;
    src = src < 0.f ? 0.f : src;
    const int i0 = (int)src;
    const int i1 = i0 + ((i0 < Tn - 1) ? 1 : 0);
    const float l1 = src - (float)i0, l0 = 1.0f - l1;
    const uint4 ua = __ldg(reinterpret_cast<const uint4*>(x + (b * Tn + i0) * hwc + e));
    const uint4 uc = __ldg(reinterpret_cast<const uint4*>(x + (b * Tn + i1) * hwc + e));
    const __nv_bfloat162* pa = reinterpret_cast<const __nv_bfloat162*>(&ua);
    const __nv_bfloat162* pc = reinterpret_cast<const __nv_bfloat162*>(&uc);
    uint4 uo;
    __nv_bfloat162* po = reinterpret_cast<__nv_bfloat162*>(&uo);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 fa = __bfloat1622float2(pa[k]), fc = __bfloat1622float2(pc[k]);
      po[k] = __floats2bfloat162_rn(__fadd_rn(__fmul_rn(l0, fa.x), __fmul_rn(l1, fc.x)), __fadd_rn(__fmul_rn(l0, fa.y), __fmul_rn(l1, fc.y)));
    }
    *reinterpret_cast<uint4*>(y + (b * 2 * Tn + j) * hwc + e) = uo;
  }
}
// split rows: row = one position (2*C bf16); interpolate hi + lo in fp32 and re-split
__global__ void __launch_bounds__(256) time_interp2x_split_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int B, int Tn,
                                                                  long long hw, int C) {
  const int c8 = C / 8;
  const long long total = (long long)B * 2 * Tn * hw * c8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % c8) * 8;
    long long r = i / c8;
    const long long pos = r % hw; r /= hw;
    const int j = (int)(r % (2 * Tn));
    const long long b = r / (2 * Tn);
    float src = 0.5f * ((float)j + 0.5f) - 0.5f;
    src = src < 0.f ? 0.f : src;
    const int i0 = (int)src;
    const int i1 = i0 + ((i0 < Tn - 1) ? 1 : 0);
    const float l1 = src - (float)i0, l0 = 1.0f - l1;
    const bf16* r0 = x + ((b * Tn + i0) * hw + pos) * 2 * C;
    const bf16* r1 = x + ((b * Tn + i1) * hw + pos) * 2 * C;
    float a[8], d[8], o[8];
    join8(*reinterpret_cast<const uint4*>(r0 + c), *reinterpret_cast<const uint4*>(r0 + C + c), a);
    join8(*reinterpret_cast<const uint4*>(r1 + c), *reinterpret_cast<const uint4*>(r1 + C + c), d);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = __fadd_rn(__fmul_rn(l0, a[k]), __fmul_rn(l1, d[k]));
    uint4 hi, lo;
    split8(o, hi, lo);
    bf16* yr = y + ((b * 2 * Tn + j) * hw + pos) * 2 * C;
    *reinterpret_cast<uint4*>(yr + c) = hi;
    *reinterpret_cast<uint4*>(yr + C + c) = lo;
  }
}
// x [batch][rows][hi(cols) | lo(cols)] -> y [batch][cols][hi(rows) | lo(rows)]
__global__ void __launch_bounds__(256) transpose_split_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int rows, int cols) {
  __shared__ bf16 tile[2][32][34];
  const bf16* xb = x + (long long)blockIdx.z * rows * cols * 2;
  bf16* yb = y + (long long)blockIdx.z * rows * cols * 2;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    tile[0][i][tx] = xb[(long long)(r0 + i) * 2 * cols + c0 + tx];
    tile[1][i][tx] = xb[(long long)(r0 + i) * 2 * cols + cols + c0 + tx];
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    yb[(long long)(c0 + i) * 2 * rows + r0 + tx] = tile[0][tx][i];
    yb[(long long)(c0 + i) * 2 * rows + rows + r0 + tx] = tile[1][tx][i];
  }
}
template <typename T>
__global__ void __launch_bounds__(256) copy_frames_kernel(const T* __restrict__ src, T* __restrict__ dst, int B,
                                                          long long src_bs, long long dst_bs, long long n) {
  const long long total = (long long)B * n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / n, e = i % n;
    dst[b * dst_bs + e] = src[b * src_bs + e];
  }
}

// 16-byte version of the two copies above / below (frame sizes, batch strides and base addresses multiples of 16 bytes --
// every cache of the model zoo): the element-wise kernels spend a 64-bit division per 2-byte element and ran at 0.8-1.5 TB/s,
// 9% + 3% of the tiled v1.1 step.
__global__ void __launch_bounds__(256) copy_frames_v16_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int B,
                                                              long long src_bs, long long dst_bs, long long n) {
  const long long total = (long long)B * n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / n, e = i - b * n;
    dst[b * dst_bs + e] = __ldg(src + b * src_bs + e);
  }
}
__global__ void __launch_bounds__(256) cache_update_v16_kernel(const uint4* __restrict__ x, const uint4* __restrict__ old_cache,
                                                               uint4* __restrict__ new_cache, int B, int Tc, int P, int off,
                                                               int first, long long fe, long long xbs) {
  const long long total = (long long)B * P * fe;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / fe;
    const long long e = i - r * fe;
    const int j = (int)(r % P);
    const long long b = r / P;
    const int idx = Tc - off + j;
    uint4 v;
    if (idx >= P) v = __ldg(x + b * xbs + (idx - P) * fe + e);
    else if (first) v = __ldg(x + b * xbs + e);
    else v = __ldg(old_cache + (b * P + (idx < 0 ? 0 : idx)) * fe + e);
    new_cache[i] = v;
  }
}

// nearest-neighbour upsampling (F.interpolate(mode="nearest"), model_3dcausal.py:209,269) of channels-last x
template <typename T>
__global__ void __launch_bounds__(256) upsample_nearest_kernel(const T* __restrict__ x, T* __restrict__ y, int B, int Tn,
                                                               int H, int W, int C4, int ut, int uh, int uw) {
  // C4 = C/4 vectors of 4 channels
  const long long total = (long long)B * Tn * ut * H * uh * W * uw * C4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    long long r = i / C4;
    const int w = (int)(r % (W * uw)); r /= (W * uw);
    const int h = (int)(r % (H * uh)); r /= (H * uh);
    const int t = (int)(r % (Tn * ut));
    const long long b = r / (Tn * ut);
    const long long src = ((((b * Tn + t / ut) * H + h / uh) * W + w / uw) * C4 + c) * 4;
    float v[4];
    load4(x + src, v);
    store4(y + i * 4, v);
  }
}
// external fp32 [B,C,T,H,W] -> channels-last [B,t_rep+T,H,W,C] with the first frame replicated t_rep times
// (EncoderCausal3DPadding.forward, model_3dcausal_v1_1.py:755-760)
template <typename T>
__global__ void __launch_bounds__(256) ncdhw_to_cl_kernel(const float* __restrict__ x, T* __restrict__ y, int B, int C,
                                                          int Tn, long long hw, int t_rep) {
  const long long total = (long long)B * (Tn + t_rep) * hw * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long r = i / C;
    const long long p = r % hw; r /= hw;
    int t = (int)(r % (Tn + t_rep)) - t_rep;
    const long long b = r / (Tn + t_rep);
    t = t < 0 ? 0 : t;
    RowAcc<T>::st(y + (i / C) * C * RowAcc<T>::W, C, c, x[((b * C + c) * Tn + t) * hw + p]);
  }
}
// v1.1 causal cache update (model_3dcausal_v1_1.py:159-176,216-233): with xp = [pad (P frames)][x (Tc frames)],
// new_cache[j] = xp[Tc - off + j], j in [0,P); pad = frame 0 of x (first chunk) or the old cache.
template <typename T>
__global__ void __launch_bounds__(256) cache_update_kernel(const T* __restrict__ x, const T* __restrict__ old_cache,
                                                           T* __restrict__ new_cache, int B, int Tc, int P, int off,
                                                           int first, long long fe, long long xbs) {
  const long long total = (long long)B * P * fe;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long e = i % fe;
    const long long r = i / fe;
    const int j = (int)(r % P);
    const long long b = r / P;
    const int idx = Tc - off + j;
    T v;
    if (idx >= P) v = x[b * xbs + (idx - P) * fe + e];
    else if (first) v = x[b * xbs + e];
    else v = old_cache[(b * P + (idx < 0 ? 0 : idx)) * fe + e];
    new_cache[i] = v;
  }
}

__global__ void __launch_bounds__(256) transpose_bf16_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int rows, int cols) {
  __shared__ bf16 tile[32][34];
  const bf16* xb = x + (long long)blockIdx.z * rows * cols;
  bf16* yb = y + (long long)blockIdx.z * rows * cols;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) tile[i][tx] = xb[(long long)(r0 + i) * cols + c0 + tx];
  __syncthreads();
  for (int i = ty; i < 32; i += 8) yb[(long long)(c0 + i) * rows + r0 + tx] = tile[tx][i];
}

// ---- decoder head as "tap planes": conv_out (Cin -> 3, 3x3x3) is first evaluated as ONE 1x1x1 GEMM producing, for
// every input position, the 27 x 4 per-tap partial outputs P[pos][tap*4 + co] (wgmma, input read once instead of 27
// times), then this kernel gathers the 27 shifted partials of each output position (causal zero padding in t, zero padding
// in h/w, model_3dcausal.py:162-197) and writes the fp32 [B,C,T,H,W] reconstruction, dropping the first to_off frames
// (model_3dcausal.py:883-885).
__global__ void __launch_bounds__(256) tap_planes_gather_kernel(const bf16* __restrict__ P, const float* __restrict__ bias,
                                                                float* __restrict__ out, int B, int Ti, int H, int W, int NP,
                                                                int Co, int to_off, int pt) {
  const int To = Ti - to_off;
  const long long total = (long long)B * To * H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int w = (int)(i % W);
    long long r = i / W;
    const int h = (int)(r % H); r /= H;
    const int to = (int)(r % To);
    const int b = (int)(r / To);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const int ti = to + to_off + a - pt;   // pt = 2: causal front padding; 1: symmetric (non-causal)
      if (ti < 0 || ti >= Ti) continue;
#pragma unroll
      for (int bb = 0; bb < 3; ++bb) {
        const int hh = h + bb - 1;
        if ((unsigned)hh >= (unsigned)H) continue;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int ww = w + c - 1;
          if ((unsigned)ww >= (unsigned)W) continue;
          const uint2 v = *reinterpret_cast<const uint2*>(P + ((((long long)b * Ti + ti) * H + hh) * W + ww) * NP + ((a * 3 + bb) * 3 + c) * 4);
          const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162*>(&v.x);
          const __nv_bfloat162 hi = *reinterpret_cast<const __nv_bfloat162*>(&v.y);
          acc[0] += __low2float(lo); acc[1] += __high2float(lo); acc[2] += __low2float(hi); acc[3] += __high2float(hi);
        }
      }
    }
    const long long plane = (long long)To * H * W;
    const long long o = (long long)b * Co * plane + ((long long)to * H + h) * W + w;
    for (int co = 0; co < Co; ++co) out[o + co * plane] = acc[co] + bias[co];
  }
}
__global__ void pack_w_tap_planes_kernel(const float* __restrict__ w, bf16* __restrict__ out, int Co, int Ci, int NP) {
  const long long total = (long long)NP * Ci;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ci = (int)(i % Ci), n = (int)(i / Ci);
    const int tap = n / 4, co = n % 4;
    float v = 0.f;
    if (tap < 27 && co < Co) v = w[((long long)co * Ci + ci) * 27 + tap];
    out[i] = __float2bfloat16_rn(v);
  }
}

// hi|lo split rows <-> fp32 rows (small fallbacks of the EXACT_TC mode)
__global__ void __launch_bounds__(256) split_to_f32_kernel(const split16* __restrict__ x, float* __restrict__ y, long long rows, int C) {
  const long long total = rows * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    y[i] = RowAcc<split16>::ld(x + (i / C) * 2 * C, C, (int)(i % C));
}
__global__ void __launch_bounds__(256) f32_to_split_kernel(const float* __restrict__ x, split16* __restrict__ y, long long rows, int C) {
  const long long total = rows * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    RowAcc<split16>::st(y + (i / C) * 2 * C, C, (int)(i % C), x[i]);
}

// ---- video I/O adjacent steps (scripts/inference_reconstruct.py:41-47,71-75 and :78-82,231-239) ------------------------
// decoded frames uint8 [T,Hs,Ws,3] (decord's HWC layout) -> centre-cropped, normalised clip fp32 [3,T,H,W] in [-1,1]:
// frames.float() / 255.0, then Normalize(mean .5, std .5) = (v - .5) / .5, op by op as torch evaluates them
__global__ void __launch_bounds__(256) u8_frames_to_clip_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst, int T,
                                                                int Hs, int Ws, int C, int h0, int w0, int H, int W) {
  const long long total = (long long)C * T * H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int w = (int)(i % W);
    long long r = i / W;
    const int h = (int)(r % H); r /= H;
    const int t = (int)(r % T);
    const int c = (int)(r / T);
    const float v = __fdiv_rn((float)src[(((long long)t * Hs + h0 + h) * Ws + w0 + w) * C + c], 255.0f);
    dst[i] = __fdiv_rn(__fsub_rn(v, 0.5f), 0.5f);
  }
}
// reconstruction fp32 [C,T,H,W] -> uint8 frames [T,H,W,C]: clamp(-1,1), (x+1)/2, *255, truncate (numpy astype(uint8))
__global__ void __launch_bounds__(256) clip_to_u8_frames_kernel(const float* __restrict__ src, uint8_t* __restrict__ dst, int C,
                                                                int T, int H, int W) {
  const long long total = (long long)T * H * W * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int w = (int)(r % W); r /= W;
    const int h = (int)(r % H);
    const int t = (int)(r / H);
    float v = src[(((long long)c * T + t) * H + h) * W + w];
    v = fminf(fmaxf(v, -1.0f), 1.0f);
    v = __fmul_rn(__fdiv_rn(__fadd_rn(v, 1.0f), 2.0f), 255.0f);
    dst[i] = (uint8_t)v;
  }
}

inline int grid_for(long long total, int block = 256) {
  long long g = (total + block - 1) / block;
  const long long cap = 132LL * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

cudaError_t launch_layernorm(DType t, const void* x, const float* gamma, const float* beta, void* y, long long rows,
                             int C, bool silu, bool exact, cudaStream_t s) {
  ProfScope _ps("layernorm", 0.0, 2.0 * rows * C * (double)dtype_size(t), s);
  const int wpb = 8;
  const unsigned grid = (unsigned)((rows + wpb - 1) / wpb);
  if (rows == 0) return cudaSuccess;
#define VT_LN_VEC(T, VPL)                                                                                            \
  do {                                                                                                               \
    if (silu && exact) layernorm_vec_kernel<T, VPL, true, true><<<grid, 256, 0, s>>>((const T*)x, gamma, beta, (T*)y, rows);        \
    else if (silu) layernorm_vec_kernel<T, VPL, true, false><<<grid, 256, 0, s>>>((const T*)x, gamma, beta, (T*)y, rows);           \
    else if (exact) layernorm_vec_kernel<T, VPL, false, true><<<grid, 256, 0, s>>>((const T*)x, gamma, beta, (T*)y, rows);          \
    else layernorm_vec_kernel<T, VPL, false, false><<<grid, 256, 0, s>>>((const T*)x, gamma, beta, (T*)y, rows);                    \
  } while (0)
#define VT_LN_GEN(T)                                                                                                 \
  do {                                                                                                               \
    if (silu) layernorm_gen_kernel<T, true, true><<<grid, 256, 0, s>>>((const T*)x, gamma, beta, (T*)y, rows, C);    \
    else layernorm_gen_kernel<T, false, true><<<grid, 256, 0, s>>>((const T*)x, gamma, beta, (T*)y, rows, C);        \
  } while (0)
  if (t == DT_SPLIT) {
    if (C % 8 == 0) {
      if (silu) layernorm_split_kernel<true><<<grid, 256, 0, s>>>((const bf16*)x, gamma, beta, (bf16*)y, rows, C);
      else layernorm_split_kernel<false><<<grid, 256, 0, s>>>((const bf16*)x, gamma, beta, (bf16*)y, rows, C);
    } else {
      VT_LN_GEN(split16);
    }
  } else if (t == DT_F32) {
    if (C == 128) VT_LN_VEC(float, 1);
    else if (C == 256) VT_LN_VEC(float, 2);
    else if (C == 512) VT_LN_VEC(float, 4);
    else VT_LN_GEN(float);
  } else if (C == 128 || C == 256 || C == 512) {
    const long long per_block = (C == 128) ? 8 * 2 * 4 : (C == 256 ? 8 * 4 : 8 * 2);
    long long gb = (rows + per_block - 1) / per_block;
    if (gb > 132 * 8) gb = 132 * 8;
#define VT_LN_BF(CC)                                                                                                  \
  do {                                                                                                                \
    if (silu) layernorm_bf16_kernel<CC, true><<<(unsigned)gb, 256, 0, s>>>((const bf16*)x, gamma, beta, (bf16*)y, rows); \
    else layernorm_bf16_kernel<CC, false><<<(unsigned)gb, 256, 0, s>>>((const bf16*)x, gamma, beta, (bf16*)y, rows);  \
  } while (0)
    if (C == 128) VT_LN_BF(128);
    else if (C == 256) VT_LN_BF(256);
    else VT_LN_BF(512);
#undef VT_LN_BF
  } else {
    VT_LN_GEN(bf16);
  }
#undef VT_LN_VEC
#undef VT_LN_GEN
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_groupnorm(DType t, const void* x, const float* gamma, const float* beta, void* y, long long frames,
                             long long ppf, int C, bool per_position, bool silu, bool exact, float* stats,
                             cudaStream_t s) {
  ProfScope _ps("groupnorm", 0.0, 2.0 * frames * ppf * C * (double)dtype_size(t), s);
  if (C % 32 != 0) return cudaErrorInvalidValue;
  const long long total = frames * ppf * C;
  if (total == 0) return cudaSuccess;
#define VT_GN(T)                                                                                                      \
  do {                                                                                                                \
    if (per_position) {                                                                                               \
      const int g = grid_for(frames * ppf * 32);                                                                      \
      if (silu) groupnorm_pos_kernel<T, true, true><<<g, 256, 0, s>>>((const T*)x, gamma, beta, (T*)y, frames * ppf, C); \
      else groupnorm_pos_kernel<T, false, true><<<g, 256, 0, s>>>((const T*)x, gamma, beta, (T*)y, frames * ppf, C);  \
      count_launch();                                                                                                 \
    } else {                                                                                                          \
      groupnorm_stats_kernel<T><<<(unsigned)(frames * 32), 256, 0, s>>>((const T*)x, stats, ppf, C);                  \
      const int g = grid_for(total);                                                                                  \
      if (silu) groupnorm_apply_kernel<T, true, true><<<g, 256, 0, s>>>((const T*)x, stats, gamma, beta, (T*)y, total, ppf, C); \
      else groupnorm_apply_kernel<T, false, true><<<g, 256, 0, s>>>((const T*)x, stats, gamma, beta, (T*)y, total, ppf, C);     \
      count_launch(2);                                                                                                \
    }                                                                                                                 \
  } while (0)
  (void)exact;
  if (t == DT_F32) VT_GN(float);
  else if (t == DT_SPLIT) VT_GN(split16);
  else VT_GN(bf16);
#undef VT_GN
  return cudaGetLastError();
}

cudaError_t launch_softmax_rows(DType tout, const float* S, void* P, long long rows, int N, cudaStream_t s) {
  ProfScope _ps("softmax", 0.0, (double)rows * N * (4.0 + dtype_size(tout)), s);
  if (rows == 0) return cudaSuccess;
  if (tout == DT_F32) softmax_rows_kernel<float><<<(unsigned)rows, 256, 0, s>>>(S, (float*)P, N);
  else if (tout == DT_SPLIT) softmax_rows_kernel<split16><<<(unsigned)rows, 256, 0, s>>>(S, (split16*)P, N);
  else softmax_rows_kernel<bf16><<<(unsigned)rows, 256, 0, s>>>(S, (bf16*)P, N);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_kl(const float* h, const float* noise, int zc, long long P, int B, bool sample, float* z,
                      float* kl_loss, double* scratch, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(scratch, 0, sizeof(double), s);
  if (e != cudaSuccess) return e;
  kl_kernel<<<grid_for((long long)B * zc * P), 256, 0, s>>>(h, noise, zc, P, B, sample ? 1 : 0, z, scratch);
  count_launch();
  if (kl_loss) {
    kl_finish_kernel<<<1, 1, 0, s>>>(scratch, B, kl_loss);
    count_launch();
  }
  return cudaGetLastError();
}

// fused KL (conv_out epilogue accumulates into `scratch`): clear before, finish after
cudaError_t launch_kl_clear(double* scratch, cudaStream_t s) { return cudaMemsetAsync(scratch, 0, sizeof(double), s); }
cudaError_t launch_kl_finish(const double* scratch, int B, float* kl_loss, cudaStream_t s) {
  if (!kl_loss) return cudaSuccess;
  kl_finish_kernel<<<1, 1, 0, s>>>(scratch, B, kl_loss);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_fsq(const float* h, int d, const int* levels, long long P, int B, float* codes, int* indices,
                       cudaStream_t s) {
  if (d > VT_MAX_FSQ) return cudaErrorInvalidValue;
  FsqConst c = make_fsq_const(d, levels);
  fsq_kernel<<<grid_for((long long)B * P), 256, 0, s>>>(h, c, P, B, codes, indices);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_fsq_indices_to_codes(const int* indices, int d, const int* levels, long long P, int B, float* codes,
                                        cudaStream_t s) {
  if (d > VT_MAX_FSQ) return cudaErrorInvalidValue;
  FsqConst c = make_fsq_const(d, levels);
  fsq_i2c_kernel<<<grid_for((long long)B * P), 256, 0, s>>>(indices, c, P, B, codes);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_pack_w_kn(const float* w, float* out, int Co, int Ci, int taps, cudaStream_t s) {
  pack_w_kn_kernel<<<grid_for((long long)Co * Ci * taps), 256, 0, s>>>(w, out, Co, Ci, taps);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_pack_w_collapsed(const float* w, bf16* out, int Co, int Co_pad, int Ci, int kt, int kh, int kw,
                                    const int* mt, const int* mh, const int* mw, int kt2, int kh2, int kw2, cudaStream_t s,
                                    float wscale) {
  CollapseMap cm;
  for (int i = 0; i < 3; ++i) { cm.mt[i] = i < kt ? mt[i] : -1; cm.mh[i] = i < kh ? mh[i] : -1; cm.mw[i] = i < kw ? mw[i] : -1; }
  pack_w_collapsed_kernel<<<grid_for((long long)Co_pad * kt2 * kh2 * kw2 * Ci), 256, 0, s>>>(w, out, Co, Co_pad, Ci, kt, kh, kw, cm, kt2, kh2, kw2, wscale);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_absmax(const float* w, long long n, float* out, cudaStream_t s) {
  absmax_kernel<<<1, 1024, 0, s>>>(w, n, out);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_pack_w_nk_bf16(const float* w, bf16* out, int Co, int Co_pad, int Ci, int taps, int Kpad, cudaStream_t s,
                                  float wscale) {
  pack_w_nk_bf16_kernel<<<grid_for((long long)Co_pad * Kpad), 256, 0, s>>>(w, out, Co, Co_pad, Ci, taps, Kpad, wscale);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_time_interp2x(DType t, const void* x, void* y, int B, int T, long long hw, int C, cudaStream_t s) {
  const long long hwc = hw * C;
  ProfScope _ps("time_interp2x", 0.0, 3.0 * B * T * hwc * (double)dtype_size(t), s);
  if (t == DT_SPLIT) {
    if (C % 8 != 0) return cudaErrorInvalidValue;
    const long long tot = (long long)B * 2 * T * hw * (C / 8);
    if (tot == 0) return cudaSuccess;
    time_interp2x_split_kernel<<<grid_for(tot), 256, 0, s>>>((const bf16*)x, (bf16*)y, B, T, hw, C);
    count_launch();
    return cudaGetLastError();
  }
  if (hwc % 4 != 0) return cudaErrorInvalidValue;
  const long long total = (long long)B * 2 * T * (hwc / 4);
  if (total == 0) return cudaSuccess;
  if (t == DT_F32) time_interp2x_kernel<float><<<grid_for(total), 256, 0, s>>>((const float*)x, (float*)y, B, T, hwc);
  else if (hwc % 8 == 0 && (((uintptr_t)x | (uintptr_t)y) & 15) == 0)
    time_interp2x_bf16x8_kernel<<<grid_for(total / 2), 256, 0, s>>>((const bf16*)x, (bf16*)y, B, T, hwc);
  else time_interp2x_kernel<bf16><<<grid_for(total), 256, 0, s>>>((const bf16*)x, (bf16*)y, B, T, hwc);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_tap_planes_gather(const bf16* P, const float* bias, float* out, int B, int Ti, int H, int W, int NP, int Co,
                                     int to_off, cudaStream_t s, int pt) {
  const long long total = (long long)B * (Ti - to_off) * H * W;
  if (total <= 0) return cudaSuccess;
  ProfScope _ps("tap_planes_gather", 2.0 * 27 * Co * total, (double)B * Ti * H * W * NP * 2.0 + (double)total * Co * 4.0, s);
  long long g = (total + 255) / 256;
  if (g > 132LL * 32) g = 132LL * 32;
  tap_planes_gather_kernel<<<(unsigned)g, 256, 0, s>>>(P, bias, out, B, Ti, H, W, NP, Co, to_off, pt);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_pack_w_tap_planes(const float* w, bf16* out, int Co, int Ci, int NP, cudaStream_t s) {
  pack_w_tap_planes_kernel<<<grid_for((long long)NP * Ci), 256, 0, s>>>(w, out, Co, Ci, NP);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_transpose_bf16(const bf16* x, bf16* y, int batch, int rows, int cols, cudaStream_t s, bool split) {
  if (rows % 32 != 0 || cols % 32 != 0) return cudaErrorInvalidValue;
  ProfScope _ps("transpose", 0.0, (split ? 8.0 : 4.0) * batch * rows * cols, s);
  dim3 grid(cols / 32, rows / 32, batch);
  if (split) transpose_split_kernel<<<grid, 256, 0, s>>>(x, y, rows, cols);
  else transpose_bf16_kernel<<<grid, 256, 0, s>>>(x, y, rows, cols);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_upsample_nearest(DType t, const void* x, void* y, int B, int T, int H, int W, int C, int ut, int uh,
                                    int uw, cudaStream_t s) {
  ProfScope _ps("upsample_nearest", 0.0, (double)B * T * H * W * C * dtype_size(t) * (1.0 + ut * uh * uw), s);
  if (C % 4 != 0) return cudaErrorInvalidValue;
  const long long total = (long long)B * T * ut * H * uh * W * uw * (C / 4);
  if (total == 0) return cudaSuccess;
  if (t != DT_BF16) upsample_nearest_kernel<float><<<grid_for(total), 256, 0, s>>>((const float*)x, (float*)y, B, T, H, W, C / 4, ut, uh, uw);
  else upsample_nearest_kernel<bf16><<<grid_for(total), 256, 0, s>>>((const bf16*)x, (bf16*)y, B, T, H, W, C / 4, ut, uh, uw);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_ncdhw_to_cl(DType t, const float* x, void* y, int B, int C, int T, int H, int W, int t_rep,
                               cudaStream_t s) {
  const long long total = (long long)B * (T + t_rep) * H * W * C;
  if (total == 0) return cudaSuccess;
  if (t == DT_F32) ncdhw_to_cl_kernel<float><<<grid_for(total), 256, 0, s>>>(x, (float*)y, B, C, T, (long long)H * W, t_rep);
  else if (t == DT_SPLIT) ncdhw_to_cl_kernel<split16><<<grid_for(total), 256, 0, s>>>(x, (split16*)y, B, C, T, (long long)H * W, t_rep);
  else ncdhw_to_cl_kernel<bf16><<<grid_for(total), 256, 0, s>>>(x, (bf16*)y, B, C, T, (long long)H * W, t_rep);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_cache_update(DType t, const void* x, const void* old_cache, void* new_cache, int B, int Tc, int P,
                                int off, bool first, long long frame_elems, long long x_bs, cudaStream_t s) {
  const long long total = (long long)B * P * frame_elems;
  if (total == 0) return cudaSuccess;
  ProfScope _ps("cache_update", 0.0, 2.0 * (double)total * (t != DT_BF16 ? 4.0 : 2.0), s);
  {
    const long long es = (t != DT_BF16) ? 4 : 2;
    const bool al = (((uintptr_t)x | (uintptr_t)old_cache | (uintptr_t)new_cache) & 15) == 0;
    if (al && (frame_elems * es) % 16 == 0 && (x_bs * es) % 16 == 0) {
      const long long fe16 = frame_elems * es / 16;
      cache_update_v16_kernel<<<grid_for((long long)B * P * fe16), 256, 0, s>>>((const uint4*)x, (const uint4*)old_cache, (uint4*)new_cache, B, Tc, P,
                                                                                 off, first ? 1 : 0, fe16, x_bs * es / 16);
      count_launch();
      return cudaGetLastError();
    }
  }
  if (t != DT_BF16) cache_update_kernel<float><<<grid_for(total), 256, 0, s>>>((const float*)x, (const float*)old_cache, (float*)new_cache, B, Tc, P, off, first ? 1 : 0, frame_elems, x_bs);
  else cache_update_kernel<bf16><<<grid_for(total), 256, 0, s>>>((const bf16*)x, (const bf16*)old_cache, (bf16*)new_cache, B, Tc, P, off, first ? 1 : 0, frame_elems, x_bs);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_copy_frames(DType t, const void* src, void* dst, int B, long long src_bs, long long dst_bs,
                               long long n, cudaStream_t s) {
  const long long total = (long long)B * n;
  if (total == 0) return cudaSuccess;
  ProfScope _ps("copy_frames", 0.0, 2.0 * (double)total * (t != DT_BF16 ? 4.0 : 2.0), s);
  {
    const long long es = (t != DT_BF16) ? 4 : 2;
    const bool al = (((uintptr_t)src | (uintptr_t)dst) & 15) == 0;
    if (al && (n * es) % 16 == 0 && (src_bs * es) % 16 == 0 && (dst_bs * es) % 16 == 0) {
      copy_frames_v16_kernel<<<grid_for((long long)B * (n * es / 16)), 256, 0, s>>>((const uint4*)src, (uint4*)dst, B, src_bs * es / 16, dst_bs * es / 16,
                                                                                    n * es / 16);
      count_launch();
      return cudaGetLastError();
    }
  }
  if (t != DT_BF16) copy_frames_kernel<float><<<grid_for(total), 256, 0, s>>>((const float*)src, (float*)dst, B, src_bs, dst_bs, n);
  else copy_frames_kernel<bf16><<<grid_for(total), 256, 0, s>>>((const bf16*)src, (bf16*)dst, B, src_bs, dst_bs, n);
  count_launch();
  return cudaGetLastError();
}

// One segment per blockIdx.y (a cache key of one batch slot); the blocks along x stride over it with 16-byte loads and
// stores when both ends are 16-byte aligned, and copy the remaining bytes (or a misaligned segment) one byte at a time.
__global__ void __launch_bounds__(256) slot_copy_kernel(const SlotSeg* __restrict__ segs) {
  const SlotSeg sg = segs[blockIdx.y];
  const char* src = (const char*)sg.src;
  char* dst = (char*)sg.dst;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  const unsigned long long t0 = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long done = 0;
  if ((((uintptr_t)src | (uintptr_t)dst) & 15) == 0) {
    const unsigned long long n16 = sg.bytes / 16;
    for (unsigned long long i = t0; i < n16; i += stride) ((uint4*)dst)[i] = __ldg((const uint4*)src + i);
    done = n16 * 16;
  }
  for (unsigned long long i = done + t0; i < sg.bytes; i += stride) dst[i] = src[i];
}
cudaError_t launch_slot_copy(const SlotSeg* segs, int n, unsigned long long max_bytes, unsigned long long total_bytes,
                             cudaStream_t s) {
  if (n <= 0 || max_bytes == 0) return cudaSuccess;
  ProfScope _ps("slot_copy", 0.0, 2.0 * (double)total_bytes, s);
  // enough blocks along x for the largest segment at 4 vectors per thread, at most 256
  const unsigned long long vec_blocks = (max_bytes / 16 + 1023) / 1024;
  const unsigned gx = (unsigned)std::min<unsigned long long>(std::max<unsigned long long>(vec_blocks, 1), 256);
  slot_copy_kernel<<<dim3(gx, (unsigned)n), 256, 0, s>>>(segs);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_u8_frames_to_clip(const uint8_t* src, float* dst, int T, int Hs, int Ws, int C, int h0, int w0, int H, int W,
                                    cudaStream_t s) {
  const long long total = (long long)C * T * H * W;
  if (total == 0) return cudaSuccess;
  ProfScope _ps("u8_frames_to_clip", 0.0, 5.0 * total, s);
  u8_frames_to_clip_kernel<<<grid_for(total), 256, 0, s>>>(src, dst, T, Hs, Ws, C, h0, w0, H, W);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_clip_to_u8_frames(const float* src, uint8_t* dst, int C, int T, int H, int W, cudaStream_t s) {
  const long long total = (long long)C * T * H * W;
  if (total == 0) return cudaSuccess;
  ProfScope _ps("clip_to_u8_frames", 0.0, 5.0 * total, s);
  clip_to_u8_frames_kernel<<<grid_for(total), 256, 0, s>>>(src, dst, C, T, H, W);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_split_to_f32(const bf16* x, float* y, long long rows, int C, cudaStream_t s) {
  if (rows * C == 0) return cudaSuccess;
  split_to_f32_kernel<<<grid_for(rows * C), 256, 0, s>>>((const split16*)x, y, rows, C);
  count_launch();
  return cudaGetLastError();
}
cudaError_t launch_f32_to_split(const float* x, bf16* y, long long rows, int C, cudaStream_t s) {
  if (rows * C == 0) return cudaSuccess;
  f32_to_split_kernel<<<grid_for(rows * C), 256, 0, s>>>(x, (split16*)y, rows, C);
  count_launch();
  return cudaGetLastError();
}

}  // namespace vt
