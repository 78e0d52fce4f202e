// Shared device/host definitions for the vidtok_b200 kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define VT_MAX_FSQ 8

namespace vt {

typedef __nv_bfloat16 bf16;

// ---- per-thread launch counter (vt_launch_count) -------------------------------------------------
extern thread_local long long g_launches;
inline void count_launch(int n = 1) { g_launches += n; }

// ---- optional per-launch profiler (vt_profile_start/stop): CUDA events on the launch stream around every kernel
struct ProfScope {
  int idx;
  cudaStream_t s;
  ProfScope(const char* name, double flops, double bytes, cudaStream_t stream, const char* detail = nullptr);
  ~ProfScope();
};
bool prof_enabled();

// ---- element helpers ------------------------------------------------------------------------------
__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(bf16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 from_f<bf16>(float v) { return __float2bfloat16_rn(v); }

// load 4 consecutive elements as floats (pointer must be 4-element aligned)
__device__ __forceinline__ void load4(const float* p, float (&o)[4]) {
  float4 v = *reinterpret_cast<const float4*>(p);
  o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
}
__device__ __forceinline__ void load4(const bf16* p, float (&o)[4]) {
  uint2 v = *reinterpret_cast<const uint2*>(p);
  __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&v.x);
  __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&v.y);
  o[0] = __low2float(a); o[1] = __high2float(a); o[2] = __low2float(b); o[3] = __high2float(b);
}
__device__ __forceinline__ void store4(float* p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void store4(bf16* p, const float (&v)[4]) {
  __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]);
  __nv_bfloat162 b = __floats2bfloat162_rn(v[2], v[3]);
  uint2 u;
  u.x = *reinterpret_cast<uint32_t*>(&a);
  u.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = u;
}

// x*sigmoid(x) = 0.5*x*(1 + tanh(0.5*x)): one MUFU (tanh.approx, rel. error ~2^-11) instead of ex2 + full division
__device__ __forceinline__ float silu_f(float x) {
  float t;
  const float hx = 0.5f * x;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(hx));
  return fmaf(hx, t, hx);
}
// accurate variant for the EXACT mode (expf, not the fast intrinsic)
__device__ __forceinline__ float silu_exact(float x) { return x * (1.0f / (1.0f + expf(-x))); }
// SiLU of the EXACT_TC epilogues: ex2.approx (2 ulp) and rcp.approx (1 ulp) instead of expf() and an IEEE division -- 5
// instructions instead of ~25 per element, relative error < 1e-6 for |x| < 16 (the epilogue was bound by this arithmetic)
__device__ __forceinline__ float silu_tc(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * x));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}

// ---- DT_SPLIT planes: v = hi + lo with hi = fp16(v), lo = fp16(v - hi): 11 + 11 mantissa bits, so a product of two split
// numbers that drops lo*lo is good to ~2^-21 (fp32-class).  (bf16 planes would give 8 + 8 bits: products good to 2^-17 only,
// measured 3e-4 on the latents -- too coarse for bit-exact FSQ codes.)  The planes are stored through bf16-typed pointers
// (16-bit elements; TMA and the data-movement kernels do not care), hence the reinterpretations.  Values beyond the fp16
// range saturate instead of becoming inf.
__device__ __forceinline__ float split_sat(float v) { return fminf(fmaxf(v, -65504.0f), 65504.0f); }
__device__ __forceinline__ void split_store(bf16* hi_p, bf16* lo_p, float v) {
  const __half h = __float2half_rn(split_sat(v));
  *reinterpret_cast<__half*>(hi_p) = h;
  *reinterpret_cast<__half*>(lo_p) = __float2half_rn(split_sat(v - __half2float(h)));
}
__device__ __forceinline__ float split_load(const bf16* hi_p, const bf16* lo_p) {
  return __half2float(*reinterpret_cast<const __half*>(hi_p)) + __half2float(*reinterpret_cast<const __half*>(lo_p));
}
// 4 consecutive fp16 values (8-byte aligned) as floats
__device__ __forceinline__ void load4h(const bf16* p, float (&o)[4]) {
  const uint2 v = *reinterpret_cast<const uint2*>(p);
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
  o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
}

// ---- regularizer arithmetic, shared by the stand-alone kernels (elementwise.cu) and the conv_out epilogue (conv_tc.cu) ----
// FSQ (regularizers.py:153-178): bound = tanh(z + shift) * half_l - offset, round half-to-even, code = q / half_w,
// index = sum_k (code_k * half_w_k + half_w_k) * basis_k -- fp32 op by op as torch evaluates it (no FMA contraction).
struct FsqConst {
  int d;
  float half_l[VT_MAX_FSQ], offset[VT_MAX_FSQ], shift[VT_MAX_FSQ], half_w[VT_MAX_FSQ];
  int levels[VT_MAX_FSQ], basis[VT_MAX_FSQ];
};
inline FsqConst make_fsq_const(int d, const int* levels) {
  FsqConst c;
  c.d = d;
  int basis = 1;
  for (int k = 0; k < VT_MAX_FSQ; ++k) { c.half_l[k] = c.offset[k] = c.shift[k] = c.half_w[k] = 0.f; c.levels[k] = c.basis[k] = 0; }
  for (int k = 0; k < d; ++k) {
    const int L = levels[k];
    c.levels[k] = L;
    c.basis[k] = basis;
    basis *= L;
    // regularizers.py:155-157, evaluated in fp32 like torch does for an int32 tensor times a python float
    const float half_l = ((float)(L - 1) * (float)(1.0 + 1e-3)) / 2.0f;
    const float offset = (L % 2 == 0) ? 0.5f : 0.0f;
    c.half_l[k] = half_l;
    c.offset[k] = offset;
    c.shift[k] = atanhf(offset / half_l);
    c.half_w[k] = (float)(L / 2);
  }
  return c;
}
// one channel of one token: returns the code, adds this digit's contribution to idx
__device__ __forceinline__ float fsq_code(const FsqConst& c, int k, float zv, float& idx) {
  const float t = (float)tanh((double)__fadd_rn(zv, c.shift[k]));
  const float bounded = __fsub_rn(__fmul_rn(t, c.half_l[k]), c.offset[k]);
  const float q = rintf(bounded);  // half-to-even, torch.round
  const float code = __fdiv_rn(q, c.half_w[k]);
  idx = __fadd_rn(idx, __fmul_rn(__fadd_rn(__fmul_rn(code, c.half_w[k]), c.half_w[k]), (float)c.basis[k]));
  return code;
}
// KL (distributions.py:8-18, regularizers.py:82-92): z = mean + exp(.5 * clamp(logvar)) * noise; returns the element's
// contribution mean^2 + var - 1 - logvar to the KL sum
__device__ __forceinline__ float kl_sample_one(float mean, float logvar, float noise, int sample, float& z) {
  logvar = fminf(fmaxf(logvar, -30.0f), 20.0f);
  const float stdv = expf(0.5f * logvar);
  const float var = expf(logvar);
  z = sample ? __fadd_rn(mean, __fmul_rn(stdv, noise)) : mean;
  return mean * mean + var - 1.0f - logvar;
}

// ---- generalized causal convolution geometry --------------------------------------------------------
// One struct describes every convolution on the path:
//   CausalConv3d / CausalConv1d (model_3dcausal.py:144-197), per-frame Conv2d of ResnetBlock (:296-306),
//   Downsample (:223-230, asymmetric zero pad + stride 2), Upsample (:208-212, nearest 2x folded into the
//   gather), TimeUpsampleResCausal2x (:267-273, nearest 2x in T folded), TimeDownsampleResCausal2x (:247-252),
//   the encoder's replicate front padding (:685-689) and the decoder's dropped frames (:883-885).
// Virtual input time axis (length t_rep + ut*Ti): [t_rep copies of frame 0][frames upsampled ut times].
// Output (to,ho,wo), tap (a,b,c) reads virtual coordinate
//   tv = (to + to_off)*st + a - pt ; hv = ho*sh + b - ph ; wv = wo*sw + c - pw
// tv < 0 : zero (t_mode 0), frame 0 (t_mode 1, v1.1 first chunk) or cache frame cacheT+tv (t_mode 2);
// hv/wv outside [0, uh*Hi) x [0, uw*Wi) : zero.  Source = (max(tv - t_rep,0)/ut, hv/uh, wv/uw).
struct ConvP {
  int B, Ti, Hi, Wi, Ci;
  long long isB, isT, isH, isW, isC;  // input element strides
  int To, Ho, Wo, Co;
  long long osB, osT, osH, osW, osC;  // output element strides
  int to_off;
  int kt, kh, kw, st, sh, sw;
  int pt, ph, pw;
  int ut, uh, uw;
  int t_rep;
  int t_mode;
  const void* cache;                  // [B, cacheT, Hi, Wi, Ci] channels-last, same type as input
  int cacheT;
  // epilogue: out = rb * (acc + bias) + ra * R
  const float* bias;
  int res_mode;                       // 0 none, 1 same index, 2 R[t/2] (time-upsample mix), 3 avgpool3 over R frames 2t-1..2t+1
  const void* res;
  long long rsB, rsT, rsH, rsW;       // residual element strides (channel stride 1)
  int resT;                           // residual frame count (mode 3 bounds)
  int res_t_mode;                     // mode 3 front pad: 0 zero (v1.0), 1 replicate frame 0, 2 res_cache (1 frame)
  int res_pool_off;                   // mode 3 window: frames 2t-1+off .. 2t+1+off (0: causal, front pad; 1: non-causal, zero frame behind the end)
  const void* res_cache;              // [B,1,H,W,C]
  float ra, rb;
  // activations (input, cache, residual, bf16-class output) are hi|lo split fp16 planes (DT_SPLIT): every position holds
  // 2*C bf16 values, the strides above count bf16 elements (isW = 2*Ci for a dense tensor), channel c's lo part is at c + C
  int split;
  // split mode: the packed weights were multiplied by a power of two (so that their lo plane stays in fp16's normal range);
  // the epilogue multiplies the accumulator by acc_scale = 2^-s before the bias (0 is read as 1)
  float acc_scale;
  // decode_from_indices in the producer of the decoder's conv_in (autoencoder.py:205-217, regularizers.py:180-198): the
  // "input" is the int32 token tensor [B,T,H,W] (strides as an fp32 tensor without the channel dimension, isC = 0) and
  // channel ci of a position is the FSQ code digit ((idx / basis_ci) % L_ci - L_ci/2) / (L_ci/2).  0 = off.
  int fsq_d;
  int fsq_levels[VT_MAX_FSQ];
  // epilogue: out = max(v, 0) after the bias and residual (the VGG16 feature stack of LPIPS); wgmma path only
  int relu;
};

}  // namespace vt
