// FP32-FMA implicit-GEMM convolution (the EXACT-mode kernel, and the fallback for shapes the wgmma kernel
// does not take: Cin=3 stem, Cout<=8 heads).  One kernel covers every convolution geometry of the path via
// ConvP (common.cuh).  GEMM view: M = B*To*Ho*Wo output positions, N = Cout, K = kt*kh*kw*Cin ordered
// tap-major / channel-minor; weights are pre-packed as [K][Cout] fp32.
#include <cstdio>
#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace vt {

namespace {

template <typename TIn>
__device__ __forceinline__ const TIn* gather_ptr(const ConvP& p, const TIn* __restrict__ x, int b, int to, int ho,
                                                 int wo, int a, int bb, int c) {
  int hv = ho * p.sh + bb - p.ph;
  int wv = wo * p.sw + c - p.pw;
  if ((unsigned)hv >= (unsigned)(p.Hi * p.uh) || (unsigned)wv >= (unsigned)(p.Wi * p.uw)) return nullptr;
  int hi = (p.uh == 2) ? (hv >> 1) : hv;
  int wi = (p.uw == 2) ? (wv >> 1) : wv;
  int tv = (to + p.to_off) * p.st + a - p.pt;
  if (tv < 0) {
    if (p.t_mode == 0) return nullptr;
    if (p.t_mode == 2) {
      int ct = p.cacheT + tv;
      return reinterpret_cast<const TIn*>(p.cache) +
             ((((long long)b * p.cacheT + ct) * p.Hi + hi) * p.Wi + wi) * (long long)p.Ci * ((std::is_same<TIn, bf16>::value && p.split) ? 2 : 1);
    }
    tv = 0;
  }
  int ti = tv - p.t_rep;
  ti = ti < 0 ? 0 : ti;
  if (p.ut == 2) ti >>= 1;
  if (ti >= p.Ti) return nullptr;   // zero padding behind the last frame (non-causal models: symmetric time padding)
  return x + (long long)b * p.isB + (long long)ti * p.isT + (long long)hi * p.isH + (long long)wi * p.isW;
}

// 4 (or ncount) consecutive channels starting at q; split tensors (hi | lo planes, DT_SPLIT) add the lo plane at q + C
template <typename T>
__device__ __forceinline__ void ld4s(const ConvP& p, const T* q, int C, int ncount, float (&t)[4]) {
  t[0] = t[1] = t[2] = t[3] = 0.f;
  if constexpr (std::is_same<T, bf16>::value) {
    if (p.split) {   // fp16 hi | lo planes behind the 16-bit pointer
      if (ncount == 4) {
        float u[4];
        load4h(q, t);
        load4h(q + C, u);
#pragma unroll
        for (int j = 0; j < 4; ++j) t[j] += u[j];
      } else {
        for (int j = 0; j < ncount; ++j) t[j] = split_load(q + j, q + C + j);
      }
      return;
    }
  }
  if (ncount == 4) {
    load4(q, t);
  } else {
    for (int j = 0; j < ncount; ++j) t[j] = to_f(q[j]);
  }
}

template <typename TRes>
__device__ __forceinline__ void residual4(const ConvP& p, int b, int to, int ho, int wo, int n, int ncount,
                                          float (&r)[4]) {
  const TRes* R = reinterpret_cast<const TRes*>(p.res);
  r[0] = r[1] = r[2] = r[3] = 0.f;
  if (p.res_mode == 1 || p.res_mode == 2) {
    int tr = (p.res_mode == 2) ? (to >> 1) : to;
    const TRes* q = R + (long long)b * p.rsB + (long long)tr * p.rsT + (long long)ho * p.rsH + (long long)wo * p.rsW + n;
    ld4s<TRes>(p, q, p.Co, ncount, r);
  } else if (p.res_mode == 3) {
    // AvgPool3d((3,1,1), stride (2,1,1)) over [front pad 1][R]  (model_3dcausal.py:242,250)
#pragma unroll
    for (int d = -1; d <= 1; ++d) {
      int tr = 2 * to + d + p.res_pool_off;
      const TRes* q = nullptr;
      if (tr >= 0) {
        if (tr < p.resT) q = R + (long long)b * p.rsB + (long long)tr * p.rsT + (long long)ho * p.rsH + (long long)wo * p.rsW + n;
      } else if (p.res_t_mode == 1) {
        q = R + (long long)b * p.rsB + (long long)ho * p.rsH + (long long)wo * p.rsW + n;
      } else if (p.res_t_mode == 2) {
        q = reinterpret_cast<const TRes*>(p.res_cache) + (((long long)b * p.Ho + ho) * p.Wo + wo) * (long long)p.Co * ((std::is_same<TRes, bf16>::value && p.split) ? 2 : 1) + n;
      }
      if (q) {
        float t[4];
        ld4s<TRes>(p, q, p.Co, ncount, t);
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] += t[j];
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) r[j] *= (1.0f / 3.0f);
  }
}

template <typename TIn, typename TOut, typename TRes, int BM, int BN, int TM, int TN, bool VECA>
__global__ void __launch_bounds__(256) conv_simt_kernel(const ConvP p, const TIn* __restrict__ x,
                                                        const float* __restrict__ w, TOut* __restrict__ out) {
  constexpr int BK = 16;
  constexpr int NTX = BN / TN;
  constexpr int NTY = BM / TM;
  static_assert(NTX * NTY == 256, "256 threads");
  static_assert(TN == 4, "TN == 4");
  constexpr int AV = BM * (BK / 4) / 256;                 // A vectors (4 k-values) per thread
  constexpr int BV = (BK * BN / 4 + 255) / 256;           // B float4 per thread (<=1)
  static_assert(BV == 1, "B tile is at most 256 float4");

  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN];

  const int tid = threadIdx.x;
  const int tx = tid % NTX, ty = tid / NTX;
  const long long M = (long long)p.B * p.To * p.Ho * p.Wo;
  const int K = p.kt * p.kh * p.kw * p.Ci;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // decode the rows this thread gathers
  int rb[AV], rt[AV], rh[AV], rw[AV];
#pragma unroll
  for (int i = 0; i < AV; ++i) {
    int v = tid + i * 256;
    long long m = m0 + (v % BM);
    if (m < M) {
      int wo = (int)(m % p.Wo);
      long long r = m / p.Wo;
      int ho = (int)(r % p.Ho);
      r /= p.Ho;
      int to = (int)(r % p.To);
      rb[i] = (int)(r / p.To); rt[i] = to; rh[i] = ho; rw[i] = wo;
    } else {
      rb[i] = -1; rt[i] = rh[i] = rw[i] = 0;
    }
  }

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  float ra[AV][4];
  float rbv[4];
  const bool vecB = (p.Co % 4) == 0;

  auto fetch = [&](int k0) {
#pragma unroll
    for (int i = 0; i < AV; ++i) {
      int v = tid + i * 256;
      int k = k0 + (v / BM) * 4;
      ra[i][0] = ra[i][1] = ra[i][2] = ra[i][3] = 0.f;
      if (rb[i] < 0) continue;
      if (VECA) {
        if (k < K) {
          int tap = k / p.Ci, ci = k - tap * p.Ci;
          int c = tap % p.kw;
          int t2 = tap / p.kw;
          int bb = t2 % p.kh, a = t2 / p.kh;
          const TIn* q = gather_ptr<TIn>(p, x, rb[i], rt[i], rh[i], rw[i], a, bb, c);
          if (q) ld4s<TIn>(p, q + ci, p.Ci, 4, ra[i]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          int kk = k + j;
          if (kk < K) {
            int tap = kk / p.Ci, ci = kk - tap * p.Ci;
            int c = tap % p.kw;
            int t2 = tap / p.kw;
            int bb = t2 % p.kh, a = t2 / p.kh;
            const TIn* q = gather_ptr<TIn>(p, x, rb[i], rt[i], rh[i], rw[i], a, bb, c);
            if (q) {
              if (std::is_same<TIn, float>::value && p.fsq_d) {
                // token index -> code digit ci (same arithmetic as fsq_i2c_kernel)
                const int id = *reinterpret_cast<const int*>(q);
                int basis = 1;
                for (int k2 = 0; k2 < ci; ++k2) basis *= p.fsq_levels[k2];
                const int L = p.fsq_levels[ci], hw = L / 2;
                ra[i][j] = (float)((id / basis) % L - hw) / (float)hw;
              } else {
                if constexpr (std::is_same<TIn, bf16>::value) {
                  ra[i][j] = p.split ? split_load(reinterpret_cast<const bf16*>(q) + (long long)ci * p.isC, reinterpret_cast<const bf16*>(q) + (long long)(ci + p.Ci) * p.isC)
                                     : to_f(q[(long long)ci * p.isC]);
                } else {
                  ra[i][j] = to_f(q[(long long)ci * p.isC]);
                }
              }
            }
          }
        }
      }
    }
    {
      int kb = tid / (BN / 4), nq = (tid % (BN / 4)) * 4;
      rbv[0] = rbv[1] = rbv[2] = rbv[3] = 0.f;
      if (tid < BK * BN / 4) {
        int k = k0 + kb, n = n0 + nq;
        if (k < K) {
          const float* q = w + (long long)k * p.Co + n;
          if (vecB && n + 3 < p.Co) {
            load4(q, rbv);
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (n + j < p.Co) rbv[j] = q[j];
          }
        }
      }
    }
  };
  auto stash = [&]() {
#pragma unroll
    for (int i = 0; i < AV; ++i) {
      int v = tid + i * 256;
      int row = v % BM, kq = (v / BM) * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) As[kq + j][row] = ra[i][j];
    }
    if (tid < BK * BN / 4) {
      int kb = tid / (BN / 4), nq = (tid % (BN / 4)) * 4;
      *reinterpret_cast<float4*>(&Bs[kb][nq]) = make_float4(rbv[0], rbv[1], rbv[2], rbv[3]);
    }
  };

  fetch(0);
  for (int k0 = 0; k0 < K; k0 += BK) {
    stash();
    __syncthreads();
    if (k0 + BK < K) fetch(k0 + BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[k][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[k][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

  // ---- epilogue: out = rb*(acc+bias) + ra*R
  const int n = n0 + tx * TN;
  if (n >= p.Co) return;
  const int ncount = (p.Co - n) >= 4 ? 4 : (p.Co - n);
  float bias[4] = {0.f, 0.f, 0.f, 0.f};
  if (p.bias)
    for (int j = 0; j < ncount; ++j) bias[j] = p.bias[n + j];
  const bool vecO = (p.osC == 1) && (p.Co % 4 == 0);
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    long long m = m0 + ty * TM + i;
    if (m >= M) continue;
    int wo = (int)(m % p.Wo);
    long long r = m / p.Wo;
    int ho = (int)(r % p.Ho);
    r /= p.Ho;
    int to = (int)(r % p.To);
    int b = (int)(r / p.To);
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = p.rb * (acc[i][j] + bias[j]);
    if (p.res_mode != 0) {
      float rr[4];
      residual4<TRes>(p, b, to, ho, wo, n, (p.Co % 4 == 0) ? 4 : ncount, rr);
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = fmaf(p.ra, rr[j], v[j]);
    }
    TOut* o = out + (long long)b * p.osB + (long long)to * p.osT + (long long)ho * p.osH + (long long)wo * p.osW +
              (long long)n * p.osC;
    if (std::is_same<TOut, bf16>::value && p.split) {
      // hi | lo planes (TOut = bf16, osC == 1)
      for (int j = 0; j < ncount; ++j) split_store(reinterpret_cast<bf16*>(o) + j, reinterpret_cast<bf16*>(o) + p.Co + j, v[j]);
    } else if (vecO) {
      store4(o, v);
    } else {
      for (int j = 0; j < ncount; ++j) o[(long long)j * p.osC] = from_f<TOut>(v[j]);
    }
  }
}

template <typename TIn, typename TOut, typename TRes>
cudaError_t launch_typed(const ConvP& p, const void* x, const float* w, void* out, cudaStream_t s) {
  const long long M = (long long)p.B * p.To * p.Ho * p.Wo;
  char det[96] = "";
  if (prof_enabled()) snprintf(det, sizeof(det), "k%d%d%d s%d%d%d u%d%d%d %d->%d @%dx%dx%d", p.kt, p.kh, p.kw, p.st, p.sh, p.sw, p.ut, p.uh, p.uw, p.Ci, p.Co, p.To, p.Ho, p.Wo);
  ProfScope _ps("conv_simt", 2.0 * M * p.kt * p.kh * p.kw * p.Ci * p.Co,
                (double)p.B * p.Ti * p.Hi * p.Wi * p.Ci * sizeof(TIn) + (double)M * p.Co * sizeof(TOut), s, det);
  const bool veca = !p.fsq_d && (p.Ci % 4 == 0) && (p.isC == 1) && (p.isW % 4 == 0) && (p.isH % 4 == 0) && (p.isT % 4 == 0) &&
                    (p.isB % 4 == 0);
  const TIn* xi = reinterpret_cast<const TIn*>(x);
  TOut* o = reinterpret_cast<TOut*>(out);
  if (p.Co <= 16) {
    constexpr int BM = 256, BN = 8;
    dim3 grid((unsigned)((M + BM - 1) / BM), (p.Co + BN - 1) / BN);
    if (veca)
      conv_simt_kernel<TIn, TOut, TRes, BM, BN, 2, 4, true><<<grid, 256, 0, s>>>(p, xi, w, o);
    else
      conv_simt_kernel<TIn, TOut, TRes, BM, BN, 2, 4, false><<<grid, 256, 0, s>>>(p, xi, w, o);
  } else {
    constexpr int BM = 64, BN = 64;
    dim3 grid((unsigned)((M + BM - 1) / BM), (p.Co + BN - 1) / BN);
    if (veca)
      conv_simt_kernel<TIn, TOut, TRes, BM, BN, 4, 4, true><<<grid, 256, 0, s>>>(p, xi, w, o);
    else
      conv_simt_kernel<TIn, TOut, TRes, BM, BN, 4, 4, false><<<grid, 256, 0, s>>>(p, xi, w, o);
  }
  count_launch();
  return cudaGetLastError();
}

}  // namespace

// DT_SPLIT tensors are 16-bit (fp16) planes behind bf16-typed pointers: the caller sets p.split when the bf16-typed operands (input / residual / output)
// are split; fp32 external tensors (tin / tout == DT_F32) are unaffected by the flag.
cudaError_t launch_conv_simt(const ConvP& p, DType tin, DType tout, DType tres, const void* x, const float* w,
                             void* out, cudaStream_t s) {
  if (tin == DT_SPLIT || tout == DT_SPLIT || tres == DT_SPLIT) {
    if (!p.split) return cudaErrorInvalidValue;
    if (tin == DT_SPLIT) tin = DT_BF16;
    if (tout == DT_SPLIT) tout = DT_BF16;
    if (tres == DT_SPLIT) tres = DT_BF16;
  } else if (p.split) {
    return cudaErrorInvalidValue;
  }
  if (tin == DT_F32 && tout == DT_F32 && tres == DT_F32) return launch_typed<float, float, float>(p, x, w, out, s);
  if (tin == DT_BF16 && tout == DT_BF16 && tres == DT_BF16) return launch_typed<bf16, bf16, bf16>(p, x, w, out, s);
  if (tin == DT_F32 && tout == DT_BF16 && tres == DT_BF16) return launch_typed<float, bf16, bf16>(p, x, w, out, s);
  if (tin == DT_BF16 && tout == DT_F32 && tres == DT_BF16) return launch_typed<bf16, float, bf16>(p, x, w, out, s);
  return cudaErrorInvalidValue;
}

// ---------------------------------------------------------------------------------------------------
// Batched strided GEMM on FP32 FMAs (attention scores / PV in EXACT mode):
//   C[z][m][n] = scale * sum_k A[z][m][k] * B[z](n,k),  B(n,k) = Bp[n*sbn + k*sbk]
// A is row-major [M][K] (lda), C row-major [M][N] (ldc).
// ---------------------------------------------------------------------------------------------------
namespace {
template <typename TA, typename TB, typename TC>
__global__ void __launch_bounds__(256) gemm_simt_kernel(const TA* __restrict__ A, const TB* __restrict__ Bm,
                                                        TC* __restrict__ C, int M, int N, int K, long long lda,
                                                        long long sbn, long long sbk, long long ldc, long long bsA,
                                                        long long bsB, long long bsC, float scale) {
  constexpr int BM = 64, BN = 64, BK = 16;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  A += (long long)blockIdx.z * bsA;
  Bm += (long long)blockIdx.z * bsB;
  C += (long long)blockIdx.z * bsC;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += BK) {
    {
      int row = tid % BM, kq = (tid / BM) * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int m = m0 + row, k = k0 + kq + j;
        As[kq + j][row] = (m < M && k < K) ? to_f(A[(long long)m * lda + k]) : 0.f;
      }
    }
    if (sbk == 1) {  // B(n,k) contiguous in k: thread reads 4 k-values of one n
      int col = tid % BN, kq = (tid / BN) * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int n = n0 + col, k = k0 + kq + j;
        Bs[kq + j][col] = (n < N && k < K) ? to_f(Bm[(long long)n * sbn + k]) : 0.f;
      }
    } else {  // contiguous in n
      int kb = tid / 16, nq = (tid % 16) * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int n = n0 + nq + j, k = k0 + kb;
        Bs[kb][nq + j] = (n < N && k < K) ? to_f(Bm[(long long)n * sbn + (long long)k * sbk]) : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int n = n0 + tx * 4 + j;
      if (n < N) C[(long long)m * ldc + n] = from_f<TC>(acc[i][j] * scale);
    }
  }
}
}  // namespace

cudaError_t launch_gemm_simt(DType ta, DType tb, DType tc, const void* A, const void* B, void* C, int M, int N, int K,
                             long long lda, long long sbn, long long sbk, long long ldc, int batch, long long bsA,
                             long long bsB, long long bsC, float scale, cudaStream_t s) {
  dim3 grid((M + 63) / 64, (N + 63) / 64, batch);
  ProfScope _ps("gemm_simt", 2.0 * M * N * K * batch, 0.0, s);
#define VT_GEMM(TA, TB, TC)                                                                                       \
  gemm_simt_kernel<TA, TB, TC><<<grid, 256, 0, s>>>((const TA*)A, (const TB*)B, (TC*)C, M, N, K, lda, sbn, sbk, ldc, \
                                                    bsA, bsB, bsC, scale)
  if (ta == DT_F32 && tb == DT_F32 && tc == DT_F32) VT_GEMM(float, float, float);
  else if (ta == DT_BF16 && tb == DT_BF16 && tc == DT_F32) VT_GEMM(bf16, bf16, float);
  else if (ta == DT_BF16 && tb == DT_BF16 && tc == DT_BF16) VT_GEMM(bf16, bf16, bf16);
  else if (ta == DT_F32 && tb == DT_BF16 && tc == DT_BF16) VT_GEMM(float, bf16, bf16);
  else return cudaErrorInvalidValue;
#undef VT_GEMM
  count_launch();
  return cudaGetLastError();
}

}  // namespace vt
