// Internal model representation: parameter manifest, packed weights, layer structure (mirrors the module
// tree of vidtok/modules/model_3dcausal.py:502-885) and the arena used by the executor.
#pragma once
#include <cuda_runtime.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/vidtok_b200.h"
#include "kernels.h"

namespace vt {

struct Param {
  std::string name;
  std::vector<int64_t> shape;
  int64_t numel = 0;
  int64_t offset = 0;  // element offset into the raw fp32 pool
  bool loaded = false;
};

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
  std::vector<vt::Param> params;
  std::map<std::string, int> index;
  float* pool = nullptr;        // raw fp32 parameters (reference layout)
  int64_t pool_elems = 0;
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
