// The parts of the FVD feature network (I3D, Inception-v1 inflated, Kinetics-400) that are not conv_tc launches: the frame
// resize and centre crop, the 7x7x7 / stride-2 stem on wgmma, the logits head and the feature statistics.  The 56 other
// convolutions run on conv_tc with the ReLU epilogue and the max-pools on maxpool3d_kernel (lpips.cu).
//
// Stem (Conv3d_1a_7x7, 3 -> 64, K = 7*7*7*3 = 1029 padded to 1088 = 17 K chunks of 64): as in conv_stem.cu the A tile is built
// by the CTA's threads, here one 64-wide K chunk at a time straight from the resized fp32 clip (L1/L2 resident: a tile's
// 128 positions read overlapping 7x7x7 windows), into a ring of three stages so that the MMAs of chunk k run while chunk
// k + 1 is gathered.  Each of the two warpgroups multiplies its 64 rows by the chunk's 64 weight rows; the epilogue adds the
// folded BatchNorm bias, applies ReLU and writes the channels-last bf16 (or hi|lo split) activation.
#include <cstdio>
#include <cstring>

#include "common.cuh"
#include "kernels.h"
#include "tc_host.h"
#include "tc_ptx.cuh"

namespace vt {
namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- resize and centre crop ----------------------------------------------------------------------------------------------
// out[g][c][t][i][j] (fp32, 224 x 224) = (bilinear(v)[i + oh][j + ow] - 0.5) * 2 with v = (clamp(x, -1, 1) + 1) / 2, the
// bilinear resize of F.interpolate(size=(Hr, Wr), mode="bilinear", align_corners=False) without antialias: source
// coordinate (d + 0.5) * in / out - 0.5, clamped at 0, each rounding step in fp32 as torch's kernel takes it.
__device__ __forceinline__ float i3d_in(const void* src, int dt, long long i) {
  float v = dt == 0 ? static_cast<const float*>(src)[i]
                    : dt == 1 ? __bfloat162float(static_cast<const bf16*>(src)[i]) : __half2float(static_cast<const __half*>(src)[i]);
  v = fminf(fmaxf(v, -1.0f), 1.0f);
  return __fdiv_rn(__fadd_rn(v, 1.0f), 2.0f);
}
__device__ __forceinline__ void src_index(int d, int in, float scale, int& i0, int& i1, float& l0, float& l1) {
  float r = __fsub_rn(__fmul_rn(scale, __fadd_rn((float)d, 0.5f)), 0.5f);
  r = r < 0.f ? 0.f : r;
  i0 = min((int)floorf(r), in - 1);
  l1 = fminf(fmaxf(__fsub_rn(r, (float)i0), 0.f), 1.f);
  l0 = __fsub_rn(1.0f, l1);
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
}

__global__ void __launch_bounds__(kThreads) i3d_resize_kernel(const void* __restrict__ x, int dt, long long n0, int G, int T, int H, int W,
                                                              int Hr, int Wr, int oh, int ow, float* __restrict__ out) {
  const long long plane = (long long)kI3dSize * kI3dSize;
  const long long total = (long long)G * 3 * T * plane;
  const float sh = (float)H / (float)Hr, sw = (float)W / (float)Wr;
  for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kThreads) {
    const int j = (int)(e % kI3dSize);
    const int i = (int)((e / kI3dSize) % kI3dSize);
    const long long f = e / plane;                // (g * 3 + c) * T + t
    const long long src_f = f + n0 * 3 * T;       // the same frame of the caller's clip n0 + g
    int h0, h1, w0, w1;
    float a0, a1, b0, b1;
    src_index(i + oh, H, sh, h0, h1, a0, a1);
    src_index(j + ow, W, sw, w0, w1, b0, b1);
    const long long base = src_f * H * W;
    const float v00 = i3d_in(x, dt, base + (long long)h0 * W + w0), v01 = i3d_in(x, dt, base + (long long)h0 * W + w1);
    const float v10 = i3d_in(x, dt, base + (long long)h1 * W + w0), v11 = i3d_in(x, dt, base + (long long)h1 * W + w1);
    const float top = __fadd_rn(__fmul_rn(v00, b0), __fmul_rn(v01, b1));
    const float bot = __fadd_rn(__fmul_rn(v10, b0), __fmul_rn(v11, b1));
    const float r = __fadd_rn(__fmul_rn(top, a0), __fmul_rn(bot, a1));
    out[e] = __fmul_rn(__fsub_rn(r, 0.5f), 2.0f);
  }
}

// ---- stem ------------------------------------------------------------------------------------------------------------------
struct I3dStemParams {
  const float* x;        // [G,3,T,224,224] fp32, the resized clips
  int T, To, Ho, Wo;
  int pt, ph, pw;        // SAME front padding
  const float* bias;     // [64], BatchNorm folded
  bf16* out;             // [G,To,Ho,Wo,64] (split: [.., hi 64 | lo 64])
  long long num_tiles;
  int tilesW, tilesH;
  float acc_scale;       // split: 2^-s of the pre-scaled weights (1 otherwise)
};
constexpr int kSBW = 16, kSBH = 8;                 // 128 output positions of one frame per tile
constexpr int kSK = 1029, kSKpad = 1088, kSKc = kSKpad / 64;
constexpr int kSStages = 3;
constexpr uint32_t kSA = 128 * 128, kSB = 64 * 128;   // one chunk: A 128 rows x 128 B, B 64 rows x 128 B (per plane)

template <bool kSplit>
__global__ void __launch_bounds__(kThreads, 1) i3d_stem_kernel(const I3dStemParams p, const bf16* __restrict__ wpk /*[64][1088] or [64][hi|lo]*/) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen = smem_raw + (base - smem_u32(smem_raw));
  constexpr uint32_t kPl = kSplit ? 2u : 1u;
  constexpr uint32_t kStage = kPl * (kSA + kSB);    // [A planes | B planes]
  int* lut = reinterpret_cast<int*>(gen + kSStages * kStage);
  float* sbias = reinterpret_cast<float*>(gen + kSStages * kStage + kSKpad * 4);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long HW = (long long)kI3dSize * kI3dSize;

  // k = tap * 3 + ci, tap = (a * 7 + b) * 7 + c (launch_pack_w_nk_bf16's order); packed (ci, a, b, c), -1 in the K padding
  for (int k = tid; k < kSKpad; k += kThreads) {
    int code = -1;
    if (k < kSK) {
      const int ci = k % 3, tap = k / 3;
      code = (ci << 12) | ((tap / 49) << 8) | (((tap / 7) % 7) << 4) | (tap % 7);
    }
    lut[k] = code;
  }
  if (tid < 64) sbias[tid] = p.bias[tid];
  __syncthreads();

  const int row = tid & 127, half = tid >> 7;
  const int g = warp >> 2, wq = warp & 3;
  // split: the tensor core's chained fp32 accumulation over all 68 K=16 steps would lose fp32-class accuracy (as conv_tc's
  // kparts), so the K chunks are summed in groups of kSGroup into acc and the groups added in order into sum
  constexpr int kSGroup = 4;
  float acc[32], sum[32];

  auto decode = [&](long long tile, int& b, int& t, int& h0, int& w0) {
    const int tw = (int)(tile % p.tilesW);
    long long m = tile / p.tilesW;
    const int th = (int)(m % p.tilesH);
    m /= p.tilesH;
    t = (int)(m % p.To);
    b = (int)(m / p.To);
    h0 = th * kSBH;
    w0 = tw * kSBW;
  };

  for (long long tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    int b, t, h0, w0;
    decode(tile, b, t, h0, w0);
    const int h = h0 + row / kSBW, w = w0 + row % kSBW;
    const bool valid = h < p.Ho && w < p.Wo;
    const int ti0 = 2 * t - p.pt, hi0 = 2 * h - p.ph, wi0 = 2 * w - p.pw;
    const float* xb = p.x + (long long)b * 3 * p.T * HW;

    for (int kc = 0; kc < kSKc; ++kc) {
      uint8_t* st = gen + (kc % kSStages) * kStage;
      // A: this thread's row, 16-byte units [4 half, 4 half + 4) of the chunk
#pragma unroll
      for (int uu = 0; uu < 4; ++uu) {
        const int u = 4 * half + uu;
        float f[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int code = lut[kc * 64 + u * 8 + e];
          float v = 0.f;
          if (valid && code >= 0) {
            const int ti = ti0 + ((code >> 8) & 15), hi = hi0 + ((code >> 4) & 15), wi = wi0 + (code & 15);
            if (ti >= 0 && ti < p.T && hi >= 0 && hi < kI3dSize && wi >= 0 && wi < kI3dSize)
              v = __ldg(xb + ((long long)(code >> 12) * p.T + ti) * HW + hi * kI3dSize + wi);
          }
          f[e] = v;
        }
        uint4 pk, pl;
        if constexpr (kSplit) {
          __half2* h2 = reinterpret_cast<__half2*>(&pk);
          __half2* l2 = reinterpret_cast<__half2*>(&pl);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            h2[e] = __floats2half2_rn(split_sat(f[2 * e]), split_sat(f[2 * e + 1]));
            const float2 hf = __half22float2(h2[e]);
            l2[e] = __floats2half2_rn(f[2 * e] - hf.x, f[2 * e + 1] - hf.y);
          }
        } else {
          __nv_bfloat162* h2 = reinterpret_cast<__nv_bfloat162*>(&pk);
#pragma unroll
          for (int e = 0; e < 4; ++e) h2[e] = __floats2bfloat162_rn(f[2 * e], f[2 * e + 1]);
        }
        *reinterpret_cast<uint4*>(st + row * 128 + ((u ^ (row & 7)) << 4)) = pk;
        if constexpr (kSplit) *reinterpret_cast<uint4*>(st + kSA + row * 128 + ((u ^ (row & 7)) << 4)) = pl;
      }
      // B: the chunk's 64 weight rows (split: hi plane, then lo plane)
      for (int i = tid; i < 64 * 8 * (int)kPl; i += kThreads) {
        const int pl = i >> 9, r = (i >> 3) & 63, u = i & 7;
        const uint4 v = *reinterpret_cast<const uint4*>(wpk + (long long)r * kSKpad * kPl + pl * kSKpad + kc * 64 + u * 8);
        *reinterpret_cast<uint4*>(st + kPl * kSA + pl * kSB + r * 128 + ((u ^ (r & 7)) << 4)) = v;
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      // every thread's part of chunk kc is written; and both warpgroups have retired the MMAs of chunk kc - 2 (the
      // wait<1> each of them passed before arriving here), so the next chunk may overwrite the stage of chunk kc - 2
      __syncthreads();
      const uint32_t sa = base + (kc % kSStages) * kStage + (uint32_t)g * 64u * 128u;
      const uint32_t sb = base + (kc % kSStages) * kStage + kPl * kSA;
      const uint32_t hi = tcx::desc_hi(1024u);
      tcx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t al = tcx::desc_lo(sa) + (uint32_t)(k * 2), bl = tcx::desc_lo(sb) + (uint32_t)(k * 2);
        const bool first = kSplit ? (kc % kSGroup == 0 && k == 0) : (kc == 0 && k == 0);
        tcx::wgmma_k16<64, kSplit>(acc, tcx::desc(al, hi), tcx::desc(bl, hi), first ? 0u : 1u);
        if constexpr (kSplit) {
          tcx::wgmma_k16<64, kSplit>(acc, tcx::desc(al + (kSA >> 4), hi), tcx::desc(bl, hi), 1u);
          tcx::wgmma_k16<64, kSplit>(acc, tcx::desc(al, hi), tcx::desc(bl + (kSB >> 4), hi), 1u);
        }
      }
      tcx::wgmma_commit();
      if (kSplit && (kc % kSGroup == kSGroup - 1 || kc == kSKc - 1)) {
        tcx::wgmma_wait<0>();
        tcx::acc_fence(acc);
#pragma unroll
        for (int i = 0; i < 32; ++i) sum[i] = kc < kSGroup ? acc[i] : sum[i] + acc[i];
      } else {
        tcx::wgmma_wait<1>();
      }
    }
    tcx::wgmma_wait<0>();
    tcx::acc_fence(acc);
    if constexpr (!kSplit) {
#pragma unroll
      for (int i = 0; i < 32; ++i) sum[i] = acc[i];
    }

    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int orow = 64 * g + 16 * wq + (lane >> 2) + 8 * r;
      const int oh = h0 + orow / kSBW, ow = w0 + orow % kSBW;
      if (oh >= p.Ho || ow >= p.Wo) continue;
      bf16* o = p.out + ((((long long)b * p.To + t) * p.Ho + oh) * p.Wo + ow) * (64 * (int)kPl);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = 8 * j + cq;
        float f0 = kSplit ? fmaf(sum[4 * j + 2 * r], p.acc_scale, sbias[c]) : sum[4 * j + 2 * r] + sbias[c];
        float f1 = kSplit ? fmaf(sum[4 * j + 2 * r + 1], p.acc_scale, sbias[c + 1]) : sum[4 * j + 2 * r + 1] + sbias[c + 1];
        f0 = f0 < 0.f ? 0.f : f0;
        f1 = f1 < 0.f ? 0.f : f1;
        if constexpr (kSplit) {
          const __half2 h2 = __floats2half2_rn(split_sat(f0), split_sat(f1));
          const float2 hf = __half22float2(h2);
          *reinterpret_cast<__half2*>(o + c) = h2;
          *reinterpret_cast<__half2*>(o + 64 + c) = __floats2half2_rn(split_sat(f0 - hf.x), split_sat(f1 - hf.y));
        } else {
          *reinterpret_cast<__nv_bfloat162*>(o + c) = __floats2bfloat162_rn(f0, f1);
        }
      }
    }
    __syncthreads();   // both warpgroups are done with the ring before the next tile's first chunks overwrite it
  }
}

// ---- head ------------------------------------------------------------------------------------------------------------------
// Block g: for each of the T5 - 1 time steps, the [2,7,7] window mean of every channel (fp32, positions in (t, h, w) order,
// then / 98), then logits[o] = bias[o] + sum_c wt[c][o] * pooled[c] in channel order; the clip's feature is the sum of its
// steps' logits / (T5 - 1).
template <bool kSplit>
__global__ void __launch_bounds__(kThreads) i3d_head_kernel(const bf16* __restrict__ f, int T5, const float* __restrict__ wt,
                                                            const float* __restrict__ bias, float* __restrict__ feat) {
  constexpr int C = kI3dFeatC, S = 7;
  constexpr long long cs = kSplit ? 2 * C : C;
  __shared__ float pooled[C];
  const int tid = threadIdx.x;
  const bf16* fc = f + (long long)blockIdx.x * T5 * S * S * cs;
  constexpr int kOut = (kI3dClasses + kThreads - 1) / kThreads;
  float sum[kOut];
#pragma unroll
  for (int q = 0; q < kOut; ++q) sum[q] = 0.f;
  for (int t = 0; t + 1 < T5; ++t) {
    for (int c = tid; c < C; c += kThreads) {
      float s = 0.f;
      for (int dt = 0; dt < 2; ++dt)
        for (int q = 0; q < S * S; ++q) {
          const bf16* e = fc + ((long long)(t + dt) * S * S + q) * cs + c;
          s += kSplit ? split_load(e, e + C) : __bfloat162float(*e);
        }
      pooled[c] = s / 98.0f;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kOut; ++q) {
      const int o = tid + q * kThreads;
      if (o < kI3dClasses) {
        float l = bias[o];
        for (int c = 0; c < C; ++c) l = fmaf(wt[(long long)c * kI3dClasses + o], pooled[c], l);
        sum[q] += l;
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int q = 0; q < kOut; ++q) {
    const int o = tid + q * kThreads;
    if (o < kI3dClasses) feat[(long long)blockIdx.x * kI3dClasses + o] = sum[q] / (float)(T5 - 1);
  }
}

// ---- statistics: stats[0] += n, stats[1 + i] += f_i, stats[401 + 400 i + j] += f_i f_j, clip by clip in index order --------
__global__ void __launch_bounds__(kThreads) i3d_stats_kernel(const float* __restrict__ feat, int G, double* __restrict__ stats) {
  constexpr int D = kI3dClasses;
  const long long e = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (e >= 1 + D + (long long)D * D) return;
  double acc = stats[e];
  if (e == 0) {
    for (int n = 0; n < G; ++n) acc += 1.0;
  } else if (e <= D) {
    for (int n = 0; n < G; ++n) acc += (double)feat[(long long)n * D + (e - 1)];
  } else {
    const int i = (int)((e - 1 - D) / D), j = (int)((e - 1 - D) % D);
    for (int n = 0; n < G; ++n) acc += (double)feat[(long long)n * D + i] * (double)feat[(long long)n * D + j];
  }
  stats[e] = acc;
}

// ---- end points: channels-last stored layout -> fp32 [N, C, T, H, W] of the real channels ---------------------------------
__global__ void __launch_bounds__(kThreads) i3d_unpack_kernel(const bf16* __restrict__ x, bool split, long long N, int T, int H, int W,
                                                              int Cs, I3dSegs segs, float* __restrict__ out) {
  const long long thw = (long long)T * H * W, total = N * segs.real * thw;
  const long long cs = split ? 2LL * Cs : (long long)Cs;
  for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < total; e += (long long)gridDim.x * kThreads) {
    const long long pos = e % thw;
    const int c = (int)((e / thw) % segs.real);
    const long long n = e / (thw * segs.real);
    int sc = c;
    for (int k = 0; k < segs.n; ++k)
      if (c >= segs.real0[k] && c < segs.real0[k] + segs.count[k]) sc = segs.stored0[k] + c - segs.real0[k];
    const bf16* v = x + (n * thw + pos) * cs + sc;
    out[e] = split ? split_load(v, v + Cs) : __bfloat162float(*v);
  }
}

unsigned grid_for(long long work) {
  long long g = (work + kThreads - 1) / kThreads;
  if (g > 132 * 16) g = 132 * 16;
  return (unsigned)(g < 1 ? 1 : g);
}

}  // namespace

cudaError_t launch_i3d_resize(const void* x, int x_dtype, long long n0, int G, int T, int H, int W, float* out, cudaStream_t s) {
  const I3dCrop c = i3d_crop(H, W);
  const long long total = (long long)G * 3 * T * kI3dSize * kI3dSize;
  ProfScope _ps("i3d_resize", 7.0 * total, (x_dtype == 0 ? 4.0 : 2.0) * G * 3 * T * H * W + 4.0 * total, s);
  i3d_resize_kernel<<<grid_for(total), kThreads, 0, s>>>(x, x_dtype, n0, G, T, H, W, c.Hr, c.Wr, c.oh, c.ow, out);
  count_launch();
  return cudaGetLastError();
}

size_t i3d_stem_smem(bool split) { return 1024 + kSStages * (split ? 2 : 1) * (kSA + kSB) + kSKpad * 4 + 64 * 4; }

cudaError_t launch_i3d_stem(const float* x, int G, int T, int To, int pt, int ph, int pw, bool split, const bf16* wpk, const float* bias,
                            float acc_scale, bf16* out, cudaStream_t s) {
  I3dStemParams t;
  memset(&t, 0, sizeof(t));
  t.x = x; t.T = T; t.To = To; t.Ho = t.Wo = kI3dSize / 2;
  t.pt = pt; t.ph = ph; t.pw = pw;
  t.bias = bias; t.out = out;
  t.acc_scale = split ? acc_scale : 1.0f;
  t.tilesW = (t.Wo + kSBW - 1) / kSBW; t.tilesH = (t.Ho + kSBH - 1) / kSBH;
  t.num_tiles = (long long)G * To * t.tilesH * t.tilesW;
  const size_t smem = i3d_stem_smem(split);
  int dev = 0;
  const cudaError_t dev_err = current_device(dev);
  if (dev_err != cudaSuccess) return dev_err;
  const int num_sms = device_sms(dev);
  const double M = (double)G * To * t.Ho * t.Wo;
  char det[96] = "";
  if (prof_enabled()) snprintf(det, sizeof(det), "k777 s222 3->64 @%dx%dx%d%s", To, t.Ho, t.Wo, split ? " split" : "");
  ProfScope _ps(split ? "i3d_stem3" : "i3d_stem", 2.0 * M * kSK * 64, 4.0 * G * 3 * T * kI3dSize * kI3dSize + M * 64 * 2.0 * (split ? 2 : 1), s, det);
  auto launch = [&](auto kern) -> cudaError_t {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    const long long slots = (long long)per_sm * num_sms;
    kern<<<(unsigned)(t.num_tiles < slots ? t.num_tiles : slots), kThreads, smem, s>>>(t, wpk);
    return cudaSuccess;
  };
  const cudaError_t e = split ? launch(i3d_stem_kernel<true>) : launch(i3d_stem_kernel<false>);
  if (e != cudaSuccess) return e;
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_i3d_head(const bf16* f, int G, int T5, bool split, const float* wt, const float* bias, float* feat, cudaStream_t s) {
  ProfScope _ps("i3d_head", (double)G * (T5 - 1) * (98.0 * kI3dFeatC + 2.0 * kI3dFeatC * kI3dClasses),
                (split ? 4.0 : 2.0) * G * T5 * 49 * kI3dFeatC + 4.0 * kI3dFeatC * kI3dClasses + 4.0 * G * kI3dClasses, s);
  if (split) i3d_head_kernel<true><<<G, kThreads, 0, s>>>(f, T5, wt, bias, feat);
  else i3d_head_kernel<false><<<G, kThreads, 0, s>>>(f, T5, wt, bias, feat);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_i3d_stats(const float* feat, int G, double* stats, cudaStream_t s) {
  const long long n = 1 + kI3dClasses + (long long)kI3dClasses * kI3dClasses;
  ProfScope _ps("i3d_stats", 2.0 * n * G, 4.0 * G * kI3dClasses + 16.0 * n, s);
  i3d_stats_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, s>>>(feat, G, stats);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_i3d_unpack(const bf16* x, bool split, long long N, int T, int H, int W, int Cs, const I3dSegs& segs, float* out,
                              cudaStream_t s) {
  const long long total = N * segs.real * T * H * W;
  ProfScope _ps("i3d_unpack", 0.0, (split ? 4.0 : 2.0) * total + 4.0 * total, s);
  i3d_unpack_kernel<<<grid_for(total), kThreads, 0, s>>>(x, split, N, T, H, W, Cs, segs, out);
  count_launch();
  return cudaGetLastError();
}

}  // namespace vt
