// Internal model representation: parameter manifest, packed weights, layer structure (mirrors the module
// tree of vidtok/modules/model_3dcausal.py:502-885) and the arena used by the executor.  Also the host helpers that the
// tokenizer (model.cu) and the evaluation networks (eval_nets.cu) share: errors, parameter sets, weight packing and the
// ConvP layout of their convolutions.
#pragma once
#include <cuda_runtime.h>

#include <cstring>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../include/vidtok_b200.h"
#include "kernels.h"

namespace vt {

// ---- errors: fail() sets the message vt_last_error returns and passes the code through ---------------------------------
int fail(int code, const char* fmt, ...);
#define VT_CUDA(call)                                                                         \
  do {                                                                                        \
    cudaError_t _e = (call);                                                                  \
    if (_e != cudaSuccess)                                                                    \
      return fail(VT_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

inline size_t align_up(size_t n, size_t a) { return (n + a - 1) / a * a; }

// Makes `device` current; VT_ERR_NO_DEVICE when no CUDA device is visible
inline int use_device(int device) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    return fail(VT_ERR_NO_DEVICE, "no CUDA device visible: vidtok_b200 has no CPU fallback");
  }
  VT_CUDA(cudaSetDevice(device));
  return VT_OK;
}

struct Param {
  std::string name;
  std::vector<int64_t> shape;
  int64_t numel = 0;
  int64_t offset = 0;  // element offset into the raw fp32 pool
  bool loaded = false;
};

// The parameters of one network under the reference's checkpoint keys, with their offsets into an fp32 pool of pool_elems
// elements.  `net` names the network in the load errors ("LPIPS ", "I3D ", or "" for the tokenizer).
struct ParamSet {
  const char* net;
  std::vector<Param> list;
  std::map<std::string, int> index;
  int64_t pool_elems = 0;
  explicit ParamSet(const char* net) : net(net) {}
  int size() const { return (int)list.size(); }
  Param& operator[](int i) { return list[i]; }
  const Param& operator[](int i) const { return list[i]; }
  int add(const std::string& name, std::vector<int64_t> shape) {
    Param p;
    p.name = name;
    p.shape = shape;
    p.numel = 1;
    for (auto s : shape) p.numel *= s;
    p.offset = pool_elems;
    pool_elems += (p.numel + 3) / 4 * 4;  // keep every tensor 16-byte aligned
    index[name] = size();
    list.push_back(p);
    return size() - 1;
  }
  // the index of parameter `name` holding numel elements; -1 after fail(VT_ERR_INVALID)
  int find(const char* name, int64_t numel) const {
    auto it = index.find(name);
    if (it == index.end()) {
      fail(VT_ERR_INVALID, "unknown %sparameter %s", net, name);
      return -1;
    }
    const Param& p = list[it->second];
    if (p.numel != numel) {
      fail(VT_ERR_INVALID, "parameter %s: expected %lld elements, got %lld", name, (long long)p.numel, (long long)numel);
      return -1;
    }
    return it->second;
  }
  int check_loaded() const {
    for (const Param& p : list)
      if (!p.loaded) return fail(VT_ERR_NOT_READY, "%sparameter %s was never loaded", net, p.name.c_str());
    return VT_OK;
  }
  // *_param_info: the shape padded with 1 to shape_len entries
  int info(int i, char* name, int cap, int64_t* shape, int shape_len, int32_t* ndim) const {
    if (i < 0 || i >= size()) return fail(VT_ERR_INVALID, "bad parameter index");
    const Param& p = list[i];
    if (name && cap > 0) {
      strncpy(name, p.name.c_str(), cap - 1);
      name[cap - 1] = 0;
    }
    if (ndim) *ndim = (int)p.shape.size();
    if (shape)
      for (size_t k = 0; k < (size_t)shape_len; ++k) shape[k] = k < p.shape.size() ? p.shape[k] : 1;
    return VT_OK;
  }
};

// ---- weight packing ------------------------------------------------------------------------------------------------------
// The power-of-two scales (split_weight_scale) of the split copies of fp32 device tensors {pointer, elements}: one max |w|
// per tensor on stream s, read back once
inline int split_weight_scales(const std::vector<std::pair<const float*, long long>>& w, float headroom, cudaStream_t s,
                               float* scale) {
  float* d_max = nullptr;
  VT_CUDA(cudaMalloc(&d_max, w.size() * sizeof(float)));
  std::vector<float> h_max(w.size());
  cudaError_t e = cudaSuccess;
  for (size_t i = 0; i < w.size() && e == cudaSuccess; ++i) e = launch_absmax(w[i].first, w[i].second, d_max + i, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(h_max.data(), d_max, h_max.size() * sizeof(float), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  cudaFree(d_max);
  if (e != cudaSuccess) return fail(VT_ERR_CUDA, "weight scales: %s", cudaGetErrorString(e));
  for (size_t i = 0; i < w.size(); ++i) scale[i] = split_weight_scale(h_max[i], headroom);
  return VT_OK;
}
// A convolution's wgmma weights from fp32 w [Co][Ci][taps]: the bf16 copy [Co_pad][Kpad] at nk, the split copy of w * wscale3
// at nk3
inline cudaError_t pack_conv_weights(const float* w, bf16* nk, bf16* nk3, int Co, int Co_pad, int Ci, int taps, int Kpad,
                                     float wscale3, cudaStream_t s) {
  const cudaError_t e = launch_pack_w_nk_bf16(w, nk, Co, Co_pad, Ci, taps, Kpad, s);
  return e == cudaSuccess ? launch_pack_w_nk_bf16(w, nk3, Co, Co_pad, Ci, taps, Kpad, s, wscale3) : e;
}

// ---- ConvP layout: every descriptor the executors and the operator entry points launch is built from these --------------
// zeroed but for the input extent, unit strides and unit upsampling
inline ConvP conv_p(int B, int Ti, int Hi, int Wi, int Ci) {
  ConvP p;
  memset(&p, 0, sizeof(p));
  p.B = B; p.Ti = Ti; p.Hi = Hi; p.Wi = Wi; p.Ci = Ci;
  p.st = p.sh = p.sw = 1; p.ut = p.uh = p.uw = 1;
  return p;
}
// element strides of one operand
struct Strides { long long B, T, H, W, C; };
// channels-last [B][T][H][W][C] with cw storage elements per channel (2 for split rows); bs >= 0 overrides the batch stride
// (views into a larger tensor)
inline Strides cl_strides(int T, int H, int W, int C, long long cw, long long bs = -1) {
  const long long sW = cw * C, sH = W * sW, sT = H * sH;
  return {bs >= 0 ? bs : T * sT, sT, sH, sW, 1};
}
inline void set_in(ConvP& p, const Strides& s) { p.isB = s.B; p.isT = s.T; p.isH = s.H; p.isW = s.W; p.isC = s.C; }
inline void set_out(ConvP& p, const Strides& s) { p.osB = s.B; p.osT = s.T; p.osH = s.H; p.osW = s.W; p.osC = s.C; }
// To / Ho / Wo from the input extent, taps, strides, upsampling and front padding already in p; pt_back, ph1, pw1: the
// padding behind the end of each axis.  False when the output is empty.
inline bool conv_out_size(ConvP& p, int pt_back, int ph1, int pw1) {
  p.To = (p.t_rep + p.ut * p.Ti + p.pt + pt_back - p.kt) / p.st + 1 - p.to_off;
  p.Ho = (p.uh * p.Hi + p.ph + ph1 - p.kh) / p.sh + 1;
  p.Wo = (p.uw * p.Wi + p.pw + pw1 - p.kw) / p.sw + 1;
  return p.To > 0 && p.Ho > 0 && p.Wo > 0;
}
// The conv_tc plan of a stride-1 convolution with bias and ReLU (LPIPS, I3D) over a channels-last input of Ci_s stored
// channels: kt x ks x ks taps, zero padding pt / pt_back in front of / behind the time axis and ps / ps_back on the spatial
// axes.  It writes Co channels of a channels-last output of out_Cs channels (a slice when out_Cs > Co: the caller offsets the
// output pointer); split: acc_scale 1 / wscale3.
inline bool relu_conv_plan(int B, int T, int H, int W, int Ci_s, int kt, int ks, int pt, int pt_back, int ps, int ps_back, int Co,
                           int out_Cs, const float* bias, float wscale3, bool split, TcPlan* pl) {
  const long long cw = split ? 2 : 1;
  ConvP p = conv_p(B, T, H, W, Ci_s);
  p.split = split ? 1 : 0;
  set_in(p, cl_strides(T, H, W, Ci_s, cw));
  p.kt = kt; p.kh = p.kw = ks;
  p.pt = pt; p.ph = p.pw = ps;
  p.Co = Co;
  conv_out_size(p, pt_back, ps_back, ps_back);
  set_out(p, cl_strides(p.To, p.Ho, p.Wo, out_Cs, cw));
  p.bias = bias;
  p.ra = 0.f; p.rb = 1.f;
  p.relu = 1;
  p.acc_scale = split ? 1.0f / wscale3 : 0.f;
  if (!conv_tc_plan(p, split ? DT_SPLIT : DT_BF16, nullptr, nullptr, 1, pl)) return false;
  if (out_Cs != Co) pl->o_lo = out_Cs;
  return true;
}

// One operator launch of the kernel the model path uses for that precision (vt_op_conv, vt_op_conv_ex, vt_op_conv_relu, ...)
int op_conv_impl(int precision, int force_simt, const vt_conv_desc* d, const vt_conv_ex* e, const void* x, const void* cache,
                 const float* w, const float* bias, const void* res, const float* gamma, const float* beta, void* out, void* out2,
                 cudaStream_t s, const TcRegFusion* reg = nullptr, bool relu = false);

struct ConvW {
  int Co = 0, Ci = 0, kt = 1, kh = 1, kw = 1;
  int pw = -1, pb = -1;      // param indices (weight, bias)
  float* w_kn = nullptr;     // [K][Co] fp32
  bf16* w_nk = nullptr;      // [Co_pad][Kpad] bf16 (wgmma B operand), may be null
  bf16* w_nk3 = nullptr;     // [Co_pad][hi(Kpad) | lo(Kpad)] fp16 planes of w * wscale3: split operand of the EXACT_TC mode
  float wscale3 = 1.f;       // power of two (kernels.h: split_weight_scale); the epilogue multiplies the accumulator by 1/wscale3
  int Kpad = 0;              // > 0: the conv has wgmma weights (Cin % 64 == 0); set with the geometry, before the weights
  int Co_pad = 0;            // Cout rounded up to 32 (zero rows)
  bool stem = false;         // the encoder's conv_in runs on conv_stem (Cin <= 4)
  bf16* w_stem = nullptr;    // [Co][128] bf16 (conv_stem.cu), only for the stem
  bf16* w_stem3 = nullptr;   // [Co][hi 128 | lo 128] (EXACT_TC)
  const float* bias = nullptr;
  int taps() const { return kt * kh * kw; }
};
struct NormW {
  int C = 0;
  int pg = -1, pb = -1;
  const float* gamma = nullptr;
  const float* beta = nullptr;
};
struct ResBlockW {           // ResnetBlock / ResnetCausalBlock1D / ResnetCausalBlock
  NormW n1, n2;
  ConvW c1, c2, nin;
  bool has_nin = false;
  std::string key;           // checkpoint prefix (identifies the causal caches in v1.1)
};
struct AttnW {
  NormW n;
  ConvW q, k, v, proj;
  std::string key;
};
struct LevelW {
  std::vector<ResBlockW> blk;   // spatial 2D blocks
  std::vector<ResBlockW> tblk;  // temporal 1D blocks
  bool has_resample = false;    // Downsample / Upsample conv
  ConvW resample;
  bool has_tres = false;        // TimeDownsampleResCausal2x / TimeUpsampleResCausal2x
  ConvW tconv;
  int p_mix = -1;
  float alpha = 0.f;            // sigmoid(mix_factor)
  int num_temp_upsample = 1;    // v1.1 decoder (model_3dcausal_v1_1.py:856,880-882)
  // phase-collapsed weights (BF16 mode): nearest-2x upsample followed by a conv == one small conv per output parity
  bool has_up_phase = false;    // spatial Upsample: 4 convs with 1x2x2 taps
  ConvW up_ph[4];
  bool has_tup_phase = false;   // v1.0 TimeUpsampleResCausal2x: 2 convs with 2x3x3 taps
  ConvW tup_ph[2];
  std::string tkey;
};
struct StackW {
  ConvW conv_in, conv_out;
  std::vector<LevelW> levels;
  ResBlockW mid1, mid2;
  AttnW attn;
  NormW norm_out;
};

struct Arena {
  char* base = nullptr;
  size_t cap = 0;
  bool dry = false;
  size_t peak = 0;
  struct Blk { size_t off, size; bool free; };
  std::vector<Blk> blks;
  void reset(void* b, size_t c, bool d);
  void* alloc(size_t n);
  void release(void* p);
};

}  // namespace vt

struct vt_model {
  vt_model_desc desc;
  int device = 0;
  vt::ParamSet params{""};
  float* pool = nullptr;        // raw fp32 parameters (reference layout)
  float* packed_kn = nullptr;   // all [K][Co] fp32 repacks
  vt::bf16* packed_nk = nullptr;
  vt::bf16* packed_nk3 = nullptr;      // split (hi|lo) copies of every wgmma weight matrix
  vt::bf16* packed_stem = nullptr;     // [Co][128] followed by the split copy [Co][256]
  vt::bf16* packed_planes = nullptr;   // decoder conv_out as 27x4 tap planes: [128][Cin] bf16
  vt::ConvW head_planes;               // 1x1x1 pseudo-conv Cin -> 128 using packed_planes
  bool finalized = false;
  vt::StackW enc, dec;
  std::vector<int> spatial_ds, tempo_ds, spatial_us, tempo_us;
  double* kl_scratch = nullptr;
  std::vector<vt::ConvW*> convs;   // every conv of both stacks (for packing)
  std::vector<vt::NormW*> norms;
  // device buffers of finished chunk states, reused by the next video (cudaMalloc/cudaFree per cache per video would
  // dominate the tiled path: ~100 caches per direction)
  std::multimap<size_t, void*> cache_pool;
  size_t cache_pool_bytes = 0;         // bytes parked in cache_pool; capped (VT_CACHE_POOL_MB, default 8192): see pool_put()
  // whole-video tiling (vt_encode_video / vt_decode_video): the library's own copy stream and the events that order chunk
  // staging (stream `copy`) against chunk compute (the caller's stream)
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_ready[2] = {nullptr, nullptr};   // staging buffer i holds its chunk           (copy -> compute)
  cudaEvent_t ev_free[2] = {nullptr, nullptr};    // the chunk that read staging buffer i is done (compute -> copy)
  cudaEvent_t ev_done[2] = {nullptr, nullptr};    // output buffer i holds its decoded chunk      (compute -> copy)
  cudaEvent_t ev_drained[2] = {nullptr, nullptr}; // output buffer i has been copied out          (copy -> compute)
  cudaEvent_t ev_join = nullptr;
};
