// Stem convolution of the encoder (conv_in: CausalConv3d(in_channels=3 -> ch, k=3), model_3dcausal.py:535,634) on
// wgmma: the input is the caller's fp32 [B,3,T,H,W] tensor, far too thin (K = 27*3 = 81) for the TMA-box
// formulation of conv_tc.cu, so the A tile is built by the CTA's threads: a halo patch of the 3 input frames is
// staged in shared memory (coalesced fp32 loads, replicate front padding and causal zero padding resolved while
// loading), every thread then writes im2col rows (81 values, bf16) straight into the canonical K-major
// SWIZZLE_128B layout (16-byte unit u of row r lives at unit u ^ (r & 7)), fences the generic->async proxy, and one
// each of the two warpgroups issues 8 wgmma (M=64 rows of the tile, N=Cout, K=128 with zero padding) into register
// accumulators.  The epilogue adds the bias and writes the bf16 channels-last activation.  The patch loads of tile i+1 are
// in flight (registers) during the MMAs and the epilogue of tile i.
#include <cstdio>
#include <cstring>

#include "common.cuh"
#include "kernels.h"
#include "tc_host.h"
#include "tc_ptx.cuh"

namespace vt {
namespace {

struct StemParams {
  const float* x;  // [B,Ci,T,H,W] fp32
  int B, Ci, T, H, W;
  int To;          // output frames = t_rep + T
  int t_rep, t_mode;
  int pt;          // front padding in time: 2 (causal) or 1 (non-causal: one zero frame on either side)
  const float* cache;   // t_mode 2: [B,Ci,2,H,W] fp32, the last two padded input frames of the previous chunk
  int Co;
  const float* bias;
  bf16* out;       // [B,To,H,W,Co]
  long long num_tiles;
  int tilesW, tilesH;
  float acc_scale;   // split: 2^-s of the pre-scaled weights (1 otherwise)
};
// LPIPS stem (kLp): a 1x3x3 convolution over To = 2 G images; image f < G is frame n0 + f of the clip x, image G + f the same
// frame of y, both [Bc,3,Tc,H,W] of dtype VT_DTYPE_* (frame n = b * Tc + t).  A kernel parameter of its own, behind the others,
// so that the encoder's instantiations keep their parameter layout and code.
struct LpStemParams {
  const void* x;
  const void* y;
  int x_dt, y_dt, G, Tc;
  long long n0;
};

// The LPIPS input of one element: the evaluation script's clamp of the reconstruction (y only), (v + 1) / 2, * 2 - 1, then
// LPIPS's ScalingLayer (v - shift) / scale, each step rounded in fp32 as torch rounds it (lpips.py:98-105)
__device__ __forceinline__ float lpips_in(const void* src, int dt, long long i, bool clamp, int c) {
  float v = dt == 0 ? static_cast<const float*>(src)[i]
                    : dt == 1 ? __bfloat162float(static_cast<const bf16*>(src)[i]) : __half2float(static_cast<const __half*>(src)[i]);
  if (clamp) v = fminf(fmaxf(v, -1.0f), 1.0f);
  v = __fdiv_rn(__fadd_rn(v, 1.0f), 2.0f);
  v = __fsub_rn(__fmul_rn(v, 2.0f), 1.0f);
  const float shift = c == 0 ? -0.030f : (c == 1 ? -0.088f : -0.188f);
  const float scale = c == 0 ? 0.458f : (c == 1 ? 0.448f : 0.450f);
  return __fdiv_rn(__fsub_rn(v, shift), scale);
}

constexpr int BW = 16, BH = 8;
constexpr int PW = BW + 2, PH = BH + 2;
constexpr int kATile = 2 * 128 * 128;  // two 64-wide K chunks of 128 rows x 128 B
constexpr int kPatchIt = 9;            // patch values per thread: Ci * 3 * PH * PW <= 4 * 540 = 2160 <= 9 * 256

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// kSplit (EXACT_TC mode): the im2col rows and the weights are hi|lo fp16 pairs, every K=16 step issues hi*hi + lo*hi +
// hi*lo into the same accumulator, and the output is written as hi | lo planes ([..., 2*Co]).
// kLp: the LPIPS stem (LpStemParams): one input frame per image, the script's preprocessing while loading, ReLU after the bias.
template <int CO, bool kSplit, bool kLp = false>
__global__ void __launch_bounds__(256, 1) conv_stem_kernel(const StemParams p, const bf16* __restrict__ wpk /*[Co][128] or [Co][hi 128 | lo 128]*/,
                                                           const LpStemParams lp) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen = smem_raw + (base - smem_u32(smem_raw));
  constexpr uint32_t kPl = kSplit ? 2u : 1u;
  // layout: A[planes] (32 KB each) | B[planes] (Co x 256 B each) | patch (Ci*3*PH*PW floats) | bias | im2col lut
  const uint32_t offA = 0, offB = kPl * kATile;
  const uint32_t offP = offB + kPl * (uint32_t)CO * 256u;
  constexpr int kTimeTaps = kLp ? 1 : 3;
  const uint32_t patch_floats = (uint32_t)p.Ci * kTimeTaps * PH * PW;
  const uint32_t offBias = offP + ((patch_floats * 4 + 15) & ~15u);
  const uint32_t offLut = offBias + 256 * 4;   // im2col k -> patch offset (or -1)
  float* patch = reinterpret_cast<float*>(gen + offP);
  float* sbias = reinterpret_cast<float*>(gen + offBias);
  int* lut = reinterpret_cast<int*>(gen + offLut);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = p.Ci * 9 * kTimeTaps;
  const int units = (K + 7) / 8;  // 16-byte units of real data per im2col row (11 for Ci = 3)

  // ---- one-time setup: zero the A tile, stage weights (swizzled) and bias
  for (uint32_t i = tid; i < kPl * kATile / 16; i += 256) reinterpret_cast<uint4*>(gen + offA)[i] = make_uint4(0, 0, 0, 0);
  for (int i = tid; i < CO * 16 * (int)kPl; i += 256) {
    const int pl = i / (CO * 16), r = i % (CO * 16);
    const int row = r >> 4, U = r & 15, kc = U >> 3, u = U & 7;
    const uint4 v = *reinterpret_cast<const uint4*>(wpk + (long long)row * 128 * kPl + pl * 128 + U * 8);
    *reinterpret_cast<uint4*>(gen + offB + pl * (CO * 256) + kc * (CO * 128) + row * 128 + ((u ^ (row & 7)) << 4)) = v;
  }
  for (int i = tid; i < CO; i += 256) sbias[i] = p.bias ? p.bias[i] : 0.f;
  if (tid < 128) {
    int off = -1;
    if (tid < K) {
      const int ci = tid % p.Ci, tap = tid / p.Ci;
      const int c = tap % 3, bb = (tap / 3) % 3, a = tap / 9;
      off = ((ci * kTimeTaps + a) * PH + bb) * PW + c;
    }
    lut[tid] = off;
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();

  auto decode = [&](long long tile, int& b, int& t, int& h0, int& w0) {
    const int tw = (int)(tile % p.tilesW);
    long long m = tile / p.tilesW;
    const int th = (int)(m % p.tilesH);
    m /= p.tilesH;
    t = (int)(m % p.To);
    b = (int)(m / p.To);
    h0 = th * BH;
    w0 = tw * BW;
  };
  // Halo patch of one tile: the global loads are issued back to back into registers (kPatchIt per thread) so that their
  // latency overlaps the MMAs and the epilogue of the previous tile; they are stored to shared memory afterwards.
  auto load_patch = [&](long long tile, float (&pv)[kPatchIt]) {
    int b, t, h0, w0;
    decode(tile, b, t, h0, w0);
    if constexpr (kLp) {
      // image t of the pass: x or y, frame n0 + t % G of the clip; zero padding outside the frame (after the scaling)
      const bool from_y = t >= lp.G;
      const long long n = lp.n0 + (from_y ? t - lp.G : t);
      const long long fb = (n / lp.Tc) * 3 * lp.Tc + n % lp.Tc;   // (b * 3 + 0) * Tc + t
      const long long plane = (long long)lp.Tc * p.H * p.W;
#pragma unroll
      for (int k = 0; k < kPatchIt; ++k) {
        const uint32_t i = (uint32_t)tid + (uint32_t)k * 256u;
        float v = 0.f;
        if (i < patch_floats) {
          const int ww = i % PW, hh = (i / PW) % PH, ci = i / (PW * PH);
          const int hv = h0 + hh - 1, wv = w0 + ww - 1;
          if (hv >= 0 && hv < p.H && wv >= 0 && wv < p.W)
            v = lpips_in(from_y ? lp.y : lp.x, from_y ? lp.y_dt : lp.x_dt, fb * p.H * p.W + ci * plane + (long long)hv * p.W + wv, from_y, ci);
        }
        pv[k] = v;
      }
      return;
    }
#pragma unroll
    for (int k = 0; k < kPatchIt; ++k) {
      const uint32_t i = (uint32_t)tid + (uint32_t)k * 256u;
      float v = 0.f;
      if (i < patch_floats) {
        const int ww = i % PW;
        uint32_t r = i / PW;
        const int hh = r % PH;
        r /= PH;
        const int a = r % 3, ci = r / 3;
        const int hv = h0 + hh - 1, wv = w0 + ww - 1;
        int tv = t + a - p.pt;  // virtual time axis: [t_rep copies of frame 0][T frames]
        bool ok = hv >= 0 && hv < p.H && wv >= 0 && wv < p.W && tv < p.t_rep + p.T;
        if (tv < 0 && p.t_mode == 2) {
          if (ok) v = p.cache[((((long long)b * p.Ci + ci) * 2 + (2 + tv)) * p.H + hv) * p.W + wv];
          ok = false;
        } else if (tv < 0) {
          if (p.t_mode == 0) ok = false;
          tv = 0;
        }
        if (ok) {
          int ti = tv - p.t_rep;
          ti = ti < 0 ? 0 : ti;
          v = p.x[((((long long)b * p.Ci + ci) * p.T + ti) * p.H + hv) * p.W + wv];
        }
      }
      pv[k] = v;
    }
  };
  auto store_patch = [&](const float (&pv)[kPatchIt]) {
#pragma unroll
    for (int k = 0; k < kPatchIt; ++k) {
      const uint32_t i = (uint32_t)tid + (uint32_t)k * 256u;
      if (i < patch_floats) patch[i] = pv[k];
    }
  };
  // im2col rows of the staged patch into the A tile (canonical K-major SWIZZLE_128B layout)
  auto im2col = [&]() {
    const int row = tid & 127, half = tid >> 7;
    const int dh = row / BW, dw = row % BW;
    const float* prow = patch + dh * PW + dw;
    uint8_t* arow = gen + offA + row * 128;
    const int u_begin = half == 0 ? 0 : (units + 1) / 2, u_end = half == 0 ? (units + 1) / 2 : units;
    for (int u = u_begin; u < u_end; ++u) {
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int off = lut[u * 8 + e];
        f[e] = off >= 0 ? prow[off] : 0.f;
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
      const int kc = u >> 3, uu = u & 7;
      *reinterpret_cast<uint4*>(arow + kc * (128 * 128) + ((uu ^ (row & 7)) << 4)) = pk;
      if constexpr (kSplit) *reinterpret_cast<uint4*>(arow + kATile + kc * (128 * 128) + ((uu ^ (row & 7)) << 4)) = pl;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  };
  // warpgroup g multiplies rows [64 g, 64 g + 64) of the A tile by the weights
  const int g = warp >> 2, wq = warp & 3;
  float acc[CO / 2];
  auto issue = [&]() {
    const uint32_t sa = base + offA + (uint32_t)g * 64u * 128u, sb = base + offB;
    const uint32_t hi = tcx::desc_hi(1024u);
    tcx::wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < 2; ++kc)
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t al = tcx::desc_lo(sa + kc * (128 * 128)) + (uint32_t)(k * 2);
        const uint32_t bl = tcx::desc_lo(sb + kc * (CO * 128)) + (uint32_t)(k * 2);
        tcx::wgmma_k16<CO, kSplit>(acc, tcx::desc(al, hi), tcx::desc(bl, hi), (kc | k) ? 1u : 0u);
        if constexpr (kSplit) {
          tcx::wgmma_k16<CO, kSplit>(acc, tcx::desc(al + (kATile >> 4), hi), tcx::desc(bl, hi), 1u);
          tcx::wgmma_k16<CO, kSplit>(acc, tcx::desc(al, hi), tcx::desc(bl + ((CO * 256) >> 4), hi), 1u);
        }
      }
    tcx::wgmma_commit();
  };
  auto epilogue = [&](long long tile) {
    int b, t, h0, w0;
    decode(tile, b, t, h0, w0);
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = 64 * g + 16 * wq + (lane >> 2) + 8 * r;
      const int h = h0 + row / BW, w = w0 + row % BW;
      if (h >= p.H || w >= p.W) continue;
      bf16* orow = p.out + ((((long long)b * p.To + t) * p.H + h) * p.W + w) * (CO * (int)kPl);
#pragma unroll
      for (int j = 0; j < CO / 8; ++j) {
        const int c = 8 * j + cq;
        if constexpr (kLp) {
          float f0 = kSplit ? fmaf(acc[4 * j + 2 * r], p.acc_scale, sbias[c]) : acc[4 * j + 2 * r] + sbias[c];
          float f1 = kSplit ? fmaf(acc[4 * j + 2 * r + 1], p.acc_scale, sbias[c + 1]) : acc[4 * j + 2 * r + 1] + sbias[c + 1];
          f0 = f0 < 0.f ? 0.f : f0;
          f1 = f1 < 0.f ? 0.f : f1;
          if constexpr (kSplit) {
            const __half2 h2 = __floats2half2_rn(split_sat(f0), split_sat(f1));
            const float2 hf = __half22float2(h2);
            *reinterpret_cast<__half2*>(orow + c) = h2;
            *reinterpret_cast<__half2*>(orow + CO + c) = __floats2half2_rn(split_sat(f0 - hf.x), split_sat(f1 - hf.y));
          } else {
            *reinterpret_cast<__nv_bfloat162*>(orow + c) = __floats2bfloat162_rn(f0, f1);
          }
        } else if constexpr (kSplit) {
          const float f0 = fmaf(acc[4 * j + 2 * r], p.acc_scale, sbias[c]);
          const float f1 = fmaf(acc[4 * j + 2 * r + 1], p.acc_scale, sbias[c + 1]);
          const __half2 h2 = __floats2half2_rn(split_sat(f0), split_sat(f1));
          const float2 hf = __half22float2(h2);
          const __half2 l2 = __floats2half2_rn(split_sat(f0 - hf.x), split_sat(f1 - hf.y));
          *reinterpret_cast<__half2*>(orow + c) = h2;
          *reinterpret_cast<__half2*>(orow + CO + c) = l2;
        } else {
          *reinterpret_cast<__nv_bfloat162*>(orow + c) =
              __floats2bfloat162_rn(acc[4 * j + 2 * r] + sbias[c], acc[4 * j + 2 * r + 1] + sbias[c + 1]);
        }
      }
    }
  };

  long long tile = blockIdx.x;
  float pv[kPatchIt];
  if (tile < p.num_tiles) {
    load_patch(tile, pv);
    store_patch(pv);
    __syncthreads();
    im2col();
    __syncthreads();
  }
  for (; tile < p.num_tiles; tile += gridDim.x) {
    const long long next = tile + gridDim.x;
    const bool has_next = next < p.num_tiles;
    issue();
    if (has_next) load_patch(next, pv);     // loads in flight across the MMAs and the epilogue
    tcx::wgmma_wait<0>();
    tcx::acc_fence(acc);
    epilogue(tile);
    __syncthreads();                        // both warpgroups are done with the A tile and the patch
    if (has_next) {
      store_patch(pv);
      __syncthreads();
      im2col();
      __syncthreads();
    }
  }
}

}  // namespace

namespace {
// new_cache[b][ci][j] = padded_input[L-2+j], padded_input = [t_rep copies of x[:,:,0]][x], L = t_rep + T >= 2
__global__ void __launch_bounds__(256) stem_cache_update_kernel(const float* __restrict__ x, float* __restrict__ cache, int B, int Ci,
                                                                int T, int t_rep, long long hw) {
  const long long total = (long long)B * Ci * 2 * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long e = i % hw;
    long long r = i / hw;
    const int j = (int)(r % 2);
    r /= 2;  // r = b*Ci + ci
    int idx = t_rep + T - 2 + j - t_rep;
    idx = idx < 0 ? 0 : idx;
    cache[i] = x[(r * T + idx) * hw + e];
  }
}
}  // namespace

cudaError_t launch_stem_cache_update(const float* x, float* cache, int B, int Ci, int T, int t_rep, int H, int W, cudaStream_t s) {
  if (t_rep + T < 2) return cudaErrorInvalidValue;
  const long long total = (long long)B * Ci * 2 * H * W;
  long long g = (total + 255) / 256;
  if (g > 132 * 8) g = 132 * 8;
  stem_cache_update_kernel<<<(unsigned)g, 256, 0, s>>>(x, cache, B, Ci, T, t_rep, (long long)H * W);
  count_launch();
  return cudaGetLastError();
}

bool conv_stem_supported(const ConvP& p) {
  if (p.kt != 3 || p.kh != 3 || p.kw != 3 || p.st != 1 || p.sh != 1 || p.sw != 1) return false;
  if (p.ut != 1 || p.uh != 1 || p.uw != 1 || p.to_off != 0 || p.res_mode != 0) return false;
  if (p.Ci * 27 > 128 || (p.Co != 64 && p.Co != 128 && p.Co != 256) || p.Co > (p.split ? 128 : 256)) return false;
  if (p.t_mode == 2 && (!p.cache || p.cacheT != 2)) return false;
  if ((p.pt != 2 && p.pt != 1) || p.ph != 1 || p.pw != 1) return false;
  if (p.pt == 1 && (p.t_mode != 0 || p.t_rep != 0)) return false;   // symmetric padding: v1.0 non-causal only
  if (p.Ho != p.Hi || p.Wo != p.Wi || p.To != p.t_rep + p.Ti) return false;
  // external NCDHW fp32 input, dense channels-last bf16 output
  if (p.isW != 1 || p.isH != p.Wi || p.isT != (long long)p.Hi * p.Wi || p.isC != p.isT * p.Ti || p.isB != p.isC * p.Ci) return false;
  const long long oc = (long long)p.Co * (p.split ? 2 : 1);
  if (p.osC != 1 || p.osW != oc || p.osH != (long long)p.Wo * oc || p.osT != p.osH * p.Ho || p.osB != p.osT * p.To) return false;
  return true;
}

// wpk: [Co][128] bf16, k = tap*Ci + ci, zero padded (launch_pack_w_nk_bf16 with Kpad = 128)
cudaError_t launch_conv_stem(const ConvP& p, const float* x, const bf16* wpk, bf16* out, cudaStream_t s) {
  StemParams t;
  t.cache = (const float*)p.cache;
  t.pt = p.pt;
  t.x = x; t.B = p.B; t.Ci = p.Ci; t.T = p.Ti; t.H = p.Hi; t.W = p.Wi; t.To = p.To; t.t_rep = p.t_rep; t.t_mode = p.t_mode;
  t.Co = p.Co; t.bias = p.bias; t.out = out;
  t.acc_scale = (p.split && p.acc_scale != 0.f) ? p.acc_scale : 1.0f;
  t.tilesW = (p.Wi + BW - 1) / BW; t.tilesH = (p.Hi + BH - 1) / BH;
  t.num_tiles = (long long)p.B * p.To * t.tilesH * t.tilesW;
  const size_t pl = p.split ? 2 : 1;
  const size_t smem = 1024 + pl * kATile + pl * (size_t)p.Co * 256 + (((size_t)p.Ci * 3 * PH * PW * 4 + 15) & ~(size_t)15) + 256 * 4 + 128 * 4;
  int dev = 0;
  const cudaError_t dev_err = current_device(dev);
  if (dev_err != cudaSuccess) return dev_err;
  const int num_sms = device_sms(dev);
  const double M = (double)t.num_tiles * 128;
  char det[96] = "";
  // plan key: " pad<front>.<back>" only for the symmetric time padding of the non-causal family
  if (prof_enabled()) snprintf(det, sizeof(det), p.pt != 2 ? "k333 %d->%d @%dx%dx%d pad%d.%d" : "k333 %d->%d @%dx%dx%d", p.Ci, p.Co, p.To,
                               p.Hi, p.Wi, p.pt, time_pad_back(p));
  ProfScope _ps(p.split ? "conv_stem3" : "conv_stem", 2.0 * M * 27 * p.Ci * p.Co, (double)p.B * p.Ci * p.Ti * p.Hi * p.Wi * 4.0 + M * p.Co * 2.0 * pl, s, det);
  // as many resident CTAs per SM as fit: the phases of a tile (patch loads -> im2col -> MMA -> epilogue) are serialised
  // inside a CTA by block barriers, and a second resident CTA fills the bubbles
  auto launch = [&](auto kern) -> cudaError_t {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    const long long slots = (long long)per_sm * num_sms;
    const unsigned grid = (unsigned)(t.num_tiles < slots ? t.num_tiles : slots);
    kern<<<grid, 256, smem, s>>>(t, wpk, LpStemParams());
    return cudaSuccess;
  };
  cudaError_t e;
  if (p.split) e = p.Co == 64 ? launch(conv_stem_kernel<64, true>) : launch(conv_stem_kernel<128, true>);
  else e = p.Co == 64 ? launch(conv_stem_kernel<64, false>) : p.Co == 128 ? launch(conv_stem_kernel<128, false>) : launch(conv_stem_kernel<256, false>);
  if (e != cudaSuccess) return e;
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_lpips_stem(const void* x, int x_dtype, const void* y, int y_dtype, int Tc, long long n0, int G, int H, int W,
                              bool split, const bf16* wpk, const float* bias, float acc_scale, bf16* out, cudaStream_t s) {
  StemParams t;
  memset(&t, 0, sizeof(t));
  LpStemParams lp;
  lp.x = x; lp.y = y; lp.x_dt = x_dtype; lp.y_dt = y_dtype; lp.Tc = Tc; lp.n0 = n0; lp.G = G;
  t.B = 1; t.Ci = 3; t.T = 2 * G; t.H = H; t.W = W; t.To = 2 * G;
  t.Co = 64; t.bias = bias; t.out = out;
  t.acc_scale = split ? acc_scale : 1.0f;
  t.tilesW = (W + BW - 1) / BW; t.tilesH = (H + BH - 1) / BH;
  t.num_tiles = (long long)t.To * t.tilesH * t.tilesW;
  const size_t pl = split ? 2 : 1;
  const size_t smem = 1024 + pl * kATile + pl * 64 * 256 + (((size_t)3 * PH * PW * 4 + 15) & ~(size_t)15) + 256 * 4 + 128 * 4;
  int dev = 0;
  const cudaError_t dev_err = current_device(dev);
  if (dev_err != cudaSuccess) return dev_err;
  const int num_sms = device_sms(dev);
  const double M = (double)2 * G * H * W;
  auto esz = [](int dt) { return dt == 0 ? 4.0 : 2.0; };
  char det[96] = "";
  if (prof_enabled()) snprintf(det, sizeof(det), "k133 3->64 @%dx%dx%d%s", 2 * G, H, W, split ? " split" : "");
  ProfScope _ps("lpips_stem", 2.0 * M * 27 * 64, (double)G * 3 * H * W * (esz(x_dtype) + esz(y_dtype)) + M * 64 * 2.0 * pl, s, det);
  auto launch = [&](auto kern) -> cudaError_t {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    const long long slots = (long long)per_sm * num_sms;
    const unsigned grid = (unsigned)(t.num_tiles < slots ? t.num_tiles : slots);
    kern<<<grid, 256, smem, s>>>(t, wpk, lp);
    return cudaSuccess;
  };
  cudaError_t e = split ? launch(conv_stem_kernel<64, true, true>) : launch(conv_stem_kernel<64, false, true>);
  if (e != cudaSuccess) return e;
  count_launch();
  return cudaGetLastError();
}

}  // namespace vt
