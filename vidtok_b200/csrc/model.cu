// Model construction (parameter manifest with the reference's checkpoint keys), weight repacking, and the
// executor that walks the encoder/decoder stacks launching the kernels.  Host-side C++; the layer order follows
// EncoderCausal3D.forward / DecoderCausal3D.forward (vidtok/modules/model_3dcausal.py:631-671,828-870) and the
// chunked v1.1 variants (vidtok/modules/model_3dcausal_v1_1.py).  Causal v1.0 models stream through the same chunk states:
// per-layer caches replace the zero front padding, and since every v1.0 norm and attention works within one frame, a
// streamed video computes the whole-clip function (bit for bit in BF16 / FMA32; see streaming.py for the split mode).
#include "model.h"

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace vt {

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
thread_local std::string g_err;
int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}
#define VT_CUDA(call)                                                                         \
  do {                                                                                        \
    cudaError_t _e = (call);                                                                  \
    if (_e != cudaSuccess)                                                                    \
      return fail(VT_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// ------------------------------------------------------------------------------------------------
// arena: first-fit allocator over the caller's workspace; `dry` mode only measures the peak
// ------------------------------------------------------------------------------------------------
static inline size_t align_up(size_t n, size_t a) { return (n + a - 1) / a * a; }
void Arena::reset(void* b, size_t c, bool d) {
  base = (char*)b;
  cap = c;
  dry = d;
  peak = 0;
  blks.clear();
  blks.push_back({0, d ? ((size_t)1 << 60) : c, true});
}
void* Arena::alloc(size_t n) {
  n = align_up(n ? n : 1, 1024);
  for (size_t i = 0; i < blks.size(); ++i) {
    if (blks[i].free && blks[i].size >= n) {
      if (blks[i].size > n) {
        Blk rest{blks[i].off + n, blks[i].size - n, true};
        blks[i].size = n;
        blks.insert(blks.begin() + i + 1, rest);
      }
      blks[i].free = false;
      peak = std::max(peak, blks[i].off + n);
      return base + blks[i].off;
    }
  }
  return nullptr;
}
void Arena::release(void* p) {
  if (!p) return;
  size_t off = (char*)p - base;
  for (size_t i = 0; i < blks.size(); ++i) {
    if (blks[i].off == off && !blks[i].free) {
      blks[i].free = true;
      if (i + 1 < blks.size() && blks[i + 1].free) {
        blks[i].size += blks[i + 1].size;
        blks.erase(blks.begin() + i + 1);
      }
      if (i > 0 && blks[i - 1].free) {
        blks[i - 1].size += blks[i].size;
        blks.erase(blks.begin() + i);
      }
      return;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// manifest
// ------------------------------------------------------------------------------------------------
static int add_param(vt_model* m, const std::string& name, std::vector<int64_t> shape) {
  Param p;
  p.name = name;
  p.shape = shape;
  p.numel = 1;
  for (auto s : shape) p.numel *= s;
  p.offset = m->pool_elems;
  m->pool_elems += (p.numel + 3) / 4 * 4;  // keep every tensor 16-byte aligned
  m->index[name] = (int)m->params.size();
  m->params.push_back(p);
  return (int)m->params.size() - 1;
}
// CausalConv3d: "<key>.conv.{weight,bias}", weight [Co,Ci,kt,kh,kw]
// (the non-causal family uses nn.Conv3d / nn.Conv1d directly: no inner ".conv", model_3dnoncausal.py:20-23,203,271,348)
static void add_conv3d(vt_model* m, ConvW& c, const std::string& key, int Co, int Ci, int k) {
  c.Co = Co; c.Ci = Ci; c.kt = c.kh = c.kw = k;
  const std::string in = m->desc.noncausal ? "" : ".conv";
  c.pw = add_param(m, key + in + ".weight", {Co, Ci, k, k, k});
  c.pb = add_param(m, key + in + ".bias", {Co});
  m->convs.push_back(&c);
}
// CausalConv1d: "<key>.conv.{weight,bias}", weight [Co,Ci,k]
static void add_conv1d(vt_model* m, ConvW& c, const std::string& key, int Co, int Ci, int k) {
  c.Co = Co; c.Ci = Ci; c.kt = k; c.kh = c.kw = 1;
  const std::string in = m->desc.noncausal ? "" : ".conv";
  c.pw = add_param(m, key + in + ".weight", {Co, Ci, k});
  c.pb = add_param(m, key + in + ".bias", {Co});
  m->convs.push_back(&c);
}
// nn.Conv2d: "<key>.{weight,bias}", weight [Co,Ci,k,k]
static void add_conv2d(vt_model* m, ConvW& c, const std::string& key, int Co, int Ci, int k) {
  c.Co = Co; c.Ci = Ci; c.kt = 1; c.kh = c.kw = k;
  c.pw = add_param(m, key + ".weight", {Co, Ci, k, k});
  c.pb = add_param(m, key + ".bias", {Co});
  m->convs.push_back(&c);
}
static void add_norm(vt_model* m, NormW& n, const std::string& key, int C) {
  n.C = C;
  const std::string k = (m->desc.norm_type == VT_NORM_LAYERNORM) ? key + ".norm" : key;
  n.pg = add_param(m, k + ".weight", {C});
  n.pb = add_param(m, k + ".bias", {C});
  m->norms.push_back(&n);
}
static void add_res2d(vt_model* m, ResBlockW& r, const std::string& key, int Ci, int Co) {
  r.key = key;
  add_norm(m, r.n1, key + ".norm1", Ci);
  add_conv2d(m, r.c1, key + ".conv1", Co, Ci, 3);
  add_norm(m, r.n2, key + ".norm2", Co);
  add_conv2d(m, r.c2, key + ".conv2", Co, Co, 3);
  r.has_nin = Ci != Co;
  if (r.has_nin) add_conv2d(m, r.nin, key + ".nin_shortcut", Co, Ci, 1);
}
static void add_res1d(vt_model* m, ResBlockW& r, const std::string& key, int C) {
  r.key = key;
  add_norm(m, r.n1, key + ".norm1", C);
  add_conv1d(m, r.c1, key + ".conv1", C, C, 3);
  add_norm(m, r.n2, key + ".norm2", C);
  add_conv1d(m, r.c2, key + ".conv2", C, C, 3);
}
static void add_res3d(vt_model* m, ResBlockW& r, const std::string& key, int C) {
  r.key = key;
  add_norm(m, r.n1, key + ".norm1", C);
  add_conv3d(m, r.c1, key + ".conv1", C, C, 3);
  add_norm(m, r.n2, key + ".norm2", C);
  add_conv3d(m, r.c2, key + ".conv2", C, C, 3);
}
static void add_attn(vt_model* m, AttnW& a, const std::string& key, int C) {
  a.key = key;
  add_norm(m, a.n, key + ".norm", C);
  add_conv3d(m, a.q, key + ".q", C, C, 1);
  add_conv3d(m, a.k, key + ".k", C, C, 1);
  add_conv3d(m, a.v, key + ".v", C, C, 1);
  add_conv3d(m, a.proj, key + ".proj_out", C, C, 1);
}
static bool contains(const std::vector<int>& v, int x) { return std::find(v.begin(), v.end(), x) != v.end(); }

// The kt x kh x kw phase conv of "nearest 2x upsample, then c" (one per output parity class)
static void phase_conv(ConvW& ph, const ConvW& c, int kt, int kh, int kw) {
  ph.Co = c.Co; ph.Ci = c.Ci; ph.kt = kt; ph.kh = kh; ph.kw = kw; ph.Co_pad = c.Co; ph.Kpad = kt * kh * kw * c.Ci;
}
// Everything the launch plans depend on is fixed with the model's geometry, so that a workspace dry run plans the same
// kernels before and after vt_model_finalize: the wgmma weight rows, the phase-collapsed upsampling convs (decoder
// Upsample / v1.0 TimeUpsampleResCausal2x), the stem kernel and the decoder head's tap planes.
static void plan_geometry(vt_model* m) {
  for (ConvW* c : m->convs) {
    c->Co_pad = (c->Co + 31) / 32 * 32;
    c->Kpad = c->Ci % 64 == 0 ? c->taps() * c->Ci : 0;
  }
  for (auto& lv : m->dec.levels) {
    lv.has_up_phase = lv.has_resample && lv.resample.Ci % 64 == 0 && lv.resample.Co % 32 == 0;
    lv.has_tup_phase = lv.has_tres && m->desc.version == 0 && lv.tconv.Ci % 64 == 0 && lv.tconv.Co % 32 == 0;
    if (lv.has_up_phase)
      for (ConvW& ph : lv.up_ph) phase_conv(ph, lv.resample, 1, 2, 2);
    if (lv.has_tup_phase)
      for (ConvW& ph : lv.tup_ph) phase_conv(ph, lv.tconv, 2, 3, 3);
  }
  ConvW& c = m->enc.conv_in;
  c.stem = c.Ci * 27 <= 128 && c.Co % 64 == 0 && c.Co <= 256 && c.kt == 3 && c.kh == 3 && c.kw == 3;
  // decoder head as tap planes (v1.0 only: zero causal padding, no chunk caches): a 1x1x1 conv Cin -> 128
  const ConvW& h = m->dec.conv_out;
  if (m->desc.version == 0 && h.kt == 3 && h.kh == 3 && h.kw == 3 && h.Co <= 4 && h.Ci % 64 == 0) {
    ConvW& hp = m->head_planes;
    hp.Co = 128; hp.Ci = h.Ci; hp.Co_pad = 128; hp.Kpad = h.Ci;
  }
}

static void build_manifest(vt_model* m) {
  const vt_model_desc& d = m->desc;
  const int L = d.num_levels;
  auto pick = [&](int n, const int32_t* arr, std::vector<int> dflt) {
    if (n < 0) return dflt;
    return std::vector<int>(arr, arr + n);
  };
  std::vector<int> dsd, dsu;
  for (int i = 0; i < L - 1; ++i) dsd.push_back(i);
  for (int i = 1; i < L; ++i) dsu.push_back(i);
  m->spatial_ds = pick(d.n_spatial_ds, d.spatial_ds, dsd);                 // model_3dcausal.py:539
  m->tempo_ds = pick(d.n_tempo_ds, d.tempo_ds, {L - 2, L - 3});            // :540
  m->spatial_us = pick(d.n_spatial_us, d.spatial_us, dsu);                 // :756
  m->tempo_us = pick(d.n_tempo_us, d.tempo_us, {1, 2});                    // :757

  // ---- encoder (model_3dcausal.py:535-620)
  StackW& e = m->enc;
  add_conv3d(m, e.conv_in, "encoder.conv_in", d.ch, d.in_channels, 3);
  e.levels.resize(L);
  int block_in = d.ch;
  for (int l = 0; l < L; ++l) {
    LevelW& lv = e.levels[l];
    const int block_out = d.ch * d.ch_mult[l];
    lv.blk.resize(d.num_res_blocks);
    lv.tblk.resize(d.num_res_blocks);
    for (int b = 0; b < d.num_res_blocks; ++b) {
      add_res2d(m, lv.blk[b], "encoder.down." + std::to_string(l) + ".block." + std::to_string(b), block_in, block_out);
      add_res1d(m, lv.tblk[b], "encoder.down_temporal." + std::to_string(l) + ".block." + std::to_string(b), block_out);
      block_in = block_out;
    }
    if (contains(m->spatial_ds, l)) {
      lv.has_resample = true;
      add_conv2d(m, lv.resample, "encoder.down." + std::to_string(l) + ".downsample.conv", block_in, block_in, 3);
      if (contains(m->tempo_ds, l)) {
        lv.has_tres = true;
        lv.tkey = "encoder.down_temporal." + std::to_string(l) + ".downsample";
        lv.p_mix = add_param(m, lv.tkey + ".mix_factor", {1});
        add_conv3d(m, lv.tconv, lv.tkey + ".conv", block_in, block_in, 3);
      }
    }
  }
  add_res3d(m, e.mid1, "encoder.mid.block_1", block_in);
  add_attn(m, e.attn, "encoder.mid.attn_1", block_in);
  add_res3d(m, e.mid2, "encoder.mid.block_2", block_in);
  add_norm(m, e.norm_out, "encoder.norm_out", block_in);
  add_conv3d(m, e.conv_out, "encoder.conv_out", d.double_z ? 2 * d.z_channels : d.z_channels, block_in, 3);

  // ---- decoder (model_3dcausal.py:724-811; v1.1 num_temp_upsample: model_3dcausal_v1_1.py:856,880-882)
  StackW& g = m->dec;
  block_in = d.ch * d.ch_mult[L - 1];
  add_conv3d(m, g.conv_in, "decoder.conv_in", block_in, d.z_channels, 3);
  add_res3d(m, g.mid1, "decoder.mid.block_1", block_in);
  add_attn(m, g.attn, "decoder.mid.attn_1", block_in);
  add_res3d(m, g.mid2, "decoder.mid.block_2", block_in);
  g.levels.resize(L);
  int ntu = 1;
  for (int l = L - 1; l >= 0; --l) {
    LevelW& lv = g.levels[l];
    const int block_out = d.ch * d.ch_mult[l];
    lv.blk.resize(d.num_res_blocks + 1);
    lv.tblk.resize(d.num_res_blocks + 1);
    for (int b = 0; b <= d.num_res_blocks; ++b) {
      add_res2d(m, lv.blk[b], "decoder.up." + std::to_string(l) + ".block." + std::to_string(b), block_in, block_out);
      add_res1d(m, lv.tblk[b], "decoder.up_temporal." + std::to_string(l) + ".block." + std::to_string(b), block_out);
      block_in = block_out;
    }
    if (contains(m->spatial_us, l)) {
      lv.has_resample = true;
      add_conv2d(m, lv.resample, "decoder.up." + std::to_string(l) + ".upsample.conv", block_in, block_in, 3);
    }
    if (contains(m->tempo_us, l)) {
      lv.has_tres = true;
      lv.tkey = "decoder.up_temporal." + std::to_string(l) + ".upsample";
      lv.p_mix = add_param(m, lv.tkey + ".mix_factor", {1});
      add_conv3d(m, lv.tconv, lv.tkey + ".conv", block_in, block_in, 3);
      lv.num_temp_upsample = ntu;
      ntu *= 2;
    }
  }
  add_norm(m, g.norm_out, "decoder.norm_out", block_in);
  add_conv3d(m, g.conv_out, "decoder.conv_out", d.out_ch, block_in, 3);
  plan_geometry(m);
}

// ------------------------------------------------------------------------------------------------
// executor
// ------------------------------------------------------------------------------------------------
struct Act {
  void* p = nullptr;
  int B = 0, T = 0, H = 0, W = 0, C = 0;
  bool owned = false;            // allocated from the arena
  long long elems() const { return (long long)B * T * H * W * C; }
  long long frame() const { return (long long)H * W * C; }
};

// A per-layer chunk cache, double-buffered: a chunk reads what the previous chunk left and writes its own tail for the next.
struct CacheBuf {
  void* buf[2] = {nullptr, nullptr};
  int cur = 0;
  size_t bytes = 0;
  bool valid = false;
  void* in() const { return buf[cur]; }         // the previous chunk's tail, read by this chunk
  void* out() const { return buf[cur ^ 1]; }    // this chunk's tail, read by the next chunk
  void commit() { cur ^= 1; valid = true; }
};

}  // namespace vt

namespace vt {
// Finished cache buffers are parked for the next video of the same geometry.  The pool is bounded: a process that tiles videos
// of many different resolutions would otherwise keep every size it has ever seen (memory torch's allocator cannot see).
static size_t cache_pool_cap() {
  static size_t cap = 0;
  if (!cap) { const char* e = getenv("VT_CACHE_POOL_MB"); cap = (size_t)(e ? atoll(e) : 8192) << 20; if (!cap) cap = 1; }
  return cap;
}
static void pool_put(vt_model* m, size_t bytes, void* ptr) {
  m->cache_pool.insert({bytes, ptr});
  m->cache_pool_bytes += bytes;
  while (m->cache_pool_bytes > cache_pool_cap() && !m->cache_pool.empty()) {   // evict the largest buffers first
    auto it = std::prev(m->cache_pool.end());
    cudaFree(it->second);
    m->cache_pool_bytes -= it->first;
    m->cache_pool.erase(it);
  }
}
static void* pool_take(vt_model* m, size_t bytes) {
  auto it = m->cache_pool.find(bytes);
  if (it == m->cache_pool.end()) return nullptr;
  void* ptr = it->second;
  m->cache_pool_bytes -= it->first;
  m->cache_pool.erase(it);
  return ptr;
}
}  // namespace vt

struct vt_chunk_state {
  vt_model* m = nullptr;
  int prec = 0;
  int B = 0, H = 0, W = 0;
  bool is_decoder = false;
  bool use_overlap = false;
  bool first = true;
  bool persist = true;           // false: one-shot "first chunk" context (untiled v1.1 forward)
  // (v1.0 streams: a persistent state; the first chunk has zero padding in front, later chunks read the caches)
  std::map<std::string, vt::CacheBuf> caches;
  ~vt_chunk_state() {
    for (auto& kv : caches)
      for (int i = 0; i < 2; ++i)
        if (kv.second.buf[i]) {
          if (m && persist) vt::pool_put(m, kv.second.bytes, kv.second.buf[i]);
          else cudaFree(kv.second.buf[i]);
        }
  }
};

namespace vt {

struct ConvOpt {
  int st = 1, sh = 1, sw = 1;
  int ph0 = -1, pw0 = -1, ph1 = -1, pw1 = -1;  // -1: (k-1)/2
  int ut = 1, uh = 1, uw = 1;
  int t_rep = 0, to_off = 0;
  int pt_front = -1, pt_back = 0;  // time padding override (non-causal models); -1: causal front pad (k-1)+(1-st)
  int res_pool_off = 0;            // res_mode 3 window offset (ConvP::res_pool_off)
  int res_mode = 0;
  const Act* res = nullptr;
  long long res_bs = -1;          // residual batch stride override (views)
  float ra = 1.f, rb = 1.f;
  const float* ext_in = nullptr;  // external fp32 NCDHW input
  bool ext_in_indices = false;    // ext_in is the int32 FSQ token tensor [B,T,H,W]: codes are formed in the conv's producer
  float* ext_out = nullptr;       // external fp32 NCDHW output
  long long in_bs = -1;           // input batch stride override (views into a larger tensor)
  const char* cache_key = nullptr;  // v1.1 causal cache identity (checkpoint prefix of the conv)
  bool force_simt = false;
  void* out_view = nullptr;       // write into an existing channels-last tensor through these element strides
  long long ov_sB = 0, ov_sT = 0, ov_sH = 0, ov_sW = 0;
  // LayerNorm(+SiLU) fusion requests (BF16 wgmma path only; silently not honoured otherwise -> check fused1/fused2)
  const NormW* ln1 = nullptr;     // replace the output by act(LN(out))           (conv1 -> norm2 of a ResBlock)
  bool ln1_silu = true;
  const NormW* ln2 = nullptr;     // additionally produce act(LN(out))            (stream producer -> next block's norm1)
  bool ln2_silu = true;
  void* ln2_view = nullptr;       // with out_view: where the normalised copy goes (same strides)
  mutable bool fused1 = false, fused2 = false;
  mutable Act ln2_act;            // filled when fused2 and no view was given
  // regularizer (KL / FSQ) fused into the epilogue of an fp32 head (encoder conv_out); honoured on the wgmma path only
  const TcRegFusion* reg = nullptr;
  bool reg_only = false;          // nobody reads the head's own output (h_pre): skip its stores when the regularizer is fused
  mutable bool fused_reg = false;
};

// ---- ConvP layout: every descriptor the executor and the operator entry points launch is built from these ------------
// zeroed but for the input extent, unit strides and unit upsampling
static ConvP conv_p(int B, int Ti, int Hi, int Wi, int Ci) {
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
static Strides cl_strides(int T, int H, int W, int C, long long cw, long long bs = -1) {
  const long long sW = cw * C, sH = W * sW, sT = H * sH;
  return {bs >= 0 ? bs : T * sT, sT, sH, sW, 1};
}
// the caller's fp32 [B][C][T][H][W] tensors
static Strides ncdhw_strides(int C, int T, int H, int W) {
  const long long sT = (long long)H * W, sC = T * sT;
  return {C * sC, sT, W, 1, sC};
}
static void set_in(ConvP& p, const Strides& s) { p.isB = s.B; p.isT = s.T; p.isH = s.H; p.isW = s.W; p.isC = s.C; }
static void set_out(ConvP& p, const Strides& s) { p.osB = s.B; p.osT = s.T; p.osH = s.H; p.osW = s.W; p.osC = s.C; }
static void set_res(ConvP& p, const Strides& s) { p.rsB = s.B; p.rsT = s.T; p.rsH = s.H; p.rsW = s.W; }   // channel stride 1
// To / Ho / Wo from the input extent, taps, strides, upsampling and front padding already in p; pt_back, ph1, pw1: the
// padding behind the end of each axis.  False when the output is empty.
static bool conv_out_size(ConvP& p, int pt_back, int ph1, int pw1) {
  p.To = (p.t_rep + p.ut * p.Ti + p.pt + pt_back - p.kt) / p.st + 1 - p.to_off;
  p.Ho = (p.uh * p.Hi + p.ph + ph1 - p.kh) / p.sh + 1;
  p.Wo = (p.uw * p.Wi + p.pw + pw1 - p.kw) / p.sw + 1;
  return p.To > 0 && p.Ho > 0 && p.Wo > 0;
}
// The encoder stem on conv_stem: 3x3x3 conv_in from the caller's fp32 [B,Ci,T,H,W] tensor after t_rep copies of frame 0,
// channels-last output.  Time padding mode, cache and acc_scale are the caller's.
static ConvP stem_p(int B, int Ci, int T, int H, int W, int Co, int t_rep, bool split, const float* bias) {
  ConvP p = conv_p(B, T, H, W, Ci);
  p.split = split ? 1 : 0;
  set_in(p, ncdhw_strides(Ci, T, H, W));
  p.To = T + t_rep; p.Ho = H; p.Wo = W; p.Co = Co;
  set_out(p, cl_strides(p.To, H, W, Co, split ? 2 : 1));
  p.kt = p.kh = p.kw = 3;
  p.pt = 2; p.ph = 1; p.pw = 1; p.t_rep = t_rep;
  p.bias = bias;
  return p;
}

// effective precision of one stack: MIXED = encoder EXACT_TC, decoder BF16
static inline int stack_prec(int precision, bool decoder) {
  if (precision == VT_PREC_MIXED) return decoder ? VT_PREC_BF16 : VT_PREC_EXACT_TC;
  return precision;
}

struct Exec {
  vt_model* m;
  int prec;          // FMA32 / BF16 / EXACT_TC (never MIXED: see stack_prec)
  DType ta;          // activation storage: fp32 / bf16 / hi|lo split bf16
  bool exact;        // full-precision activations functions (everything but BF16)
  bool tcm;          // tensor-core modes (BF16, EXACT_TC)
  bool split;        // ta == DT_SPLIT
  int cw;            // storage elements per logical channel (2 for split rows)
  cudaStream_t s;
  Arena ar;
  bool dry;
  vt_chunk_state* ck = nullptr;   // v1.1 chunk context; for v1.0 only set while streaming (null: whole clip)
  int rc = VT_OK;

  Exec(vt_model* m_, int prec_, cudaStream_t s_, void* ws, size_t ws_bytes, bool dry_)
      : m(m_), prec(prec_), ta(prec_ == VT_PREC_FMA32 ? DT_F32 : (prec_ == VT_PREC_EXACT_TC ? DT_SPLIT : DT_BF16)),
        exact(prec_ != VT_PREC_BF16), tcm(prec_ != VT_PREC_FMA32), split(prec_ == VT_PREC_EXACT_TC),
        cw(prec_ == VT_PREC_EXACT_TC ? 2 : 1), s(s_), dry(dry_) {
    ar.reset(dry_ ? (void*)(uintptr_t)0x100000 : ws, ws_bytes, dry_);
  }
  bool ok() const { return rc == VT_OK; }
  bool cuda(cudaError_t e, const char* what) {
    if (e != cudaSuccess && rc == VT_OK) rc = fail(VT_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
    return e == cudaSuccess;
  }
  void* alloc(size_t bytes) {
    if (!ok()) return nullptr;
    void* p = ar.alloc(bytes);
    if (!p) rc = fail(VT_ERR_WORKSPACE, "workspace too small: need %zu more bytes (capacity %zu)", bytes, ar.cap);
    return p;
  }
  Act new_act(int B, int T, int H, int W, int C) {
    Act a;
    a.B = B; a.T = T; a.H = H; a.W = W; a.C = C;
    a.p = alloc((size_t)a.elems() * dtype_size(ta));
    a.owned = true;
    return a;
  }
  void free_act(Act& a) {
    if (a.owned && a.p) ar.release(a.p);
    a.p = nullptr;
    a.owned = false;
  }

  // ---- v1.1 cache plumbing --------------------------------------------------------------------
  int cache_offset_for(const std::string& key) const {
    // autoencoder_v1_1.py:307-320 (tile_decode with use_overlap); longest-prefix rule
    if (!ck || !ck->is_decoder || !ck->use_overlap) return 0;
    const int tdf = m->desc.time_downsample_factor;
    struct R { const char* p; int v; };
    std::vector<R> rules;
    rules.push_back({"decoder.", 1});
    if (tdf == 4) {
      rules.push_back({"decoder.up_temporal.2.upsample", 2});
      rules.push_back({"decoder.up_temporal.1.", 2});
      rules.push_back({"decoder.up_temporal.1.upsample", 4});
      rules.push_back({"decoder.up_temporal.0.", 4});
      rules.push_back({"decoder.conv_out", 4});
    } else if (tdf == 2) {
      rules.push_back({"decoder.up_temporal.2.upsample", 2});
      rules.push_back({"decoder.up_temporal.1.", 2});
      rules.push_back({"decoder.up_temporal.0.", 2});
      rules.push_back({"decoder.conv_out", 2});
    } else if (tdf == 8) {
      rules.push_back({"decoder.up_temporal.3.upsample", 2});
      rules.push_back({"decoder.up_temporal.2.", 2});
      rules.push_back({"decoder.up_temporal.2.upsample", 4});
      rules.push_back({"decoder.up_temporal.1.", 4});
      rules.push_back({"decoder.up_temporal.1.upsample", 8});
      rules.push_back({"decoder.up_temporal.0.", 8});
      rules.push_back({"decoder.conv_out", 8});
    }
    int best = -1, val = 0;
    for (auto& r : rules) {
      const int n = (int)strlen(r.p);
      if ((int)key.size() >= n && key.compare(0, n, r.p) == 0 && n > best) { best = n; val = r.v; }
    }
    return val;
  }
  // The chunk cache under `key`, (re)allocated or taken from the pool when its size changes.  A later chunk of a real run reads
  // what the previous chunk committed: an empty cache there is VT_ERR_NOT_READY.  Null on error.
  CacheBuf* cache(const std::string& key, size_t bytes) {
    CacheBuf& c = ck->caches[key];
    if (c.bytes != bytes) {
      if (dry) { c.bytes = bytes; return &c; }
      for (int i = 0; i < 2; ++i) {
        if (c.buf[i]) pool_put(m, c.bytes, c.buf[i]);
        c.buf[i] = pool_take(m, bytes);
        if (!c.buf[i] && !cuda(cudaMalloc(&c.buf[i], bytes), "cudaMalloc(causal cache)")) return nullptr;
      }
      c.bytes = bytes; c.valid = false; c.cur = 0;
    }
    if (!dry && !ck->first && !c.valid) { rc = fail(VT_ERR_NOT_READY, "cache %s empty on a non-first chunk", key.c_str()); return nullptr; }
    return &c;
  }
  // this chunk's tail becomes the next chunk's input (a dry run leaves the caches as they are)
  void commit(CacheBuf* c) { if (c && !dry) c->commit(); }
  // streaming: caches live across chunks (v1.1 tiling, v1.0 streams)
  bool streaming() const { return ck && ck->persist; }
  // dst [rows][2][fe] := the last two frames of [front (2 frames) | x (T frames)], rows of x T * fe apart; null front: zero
  // frames (the causal padding in front of a first chunk)
  void tail2(DType t, const void* x, const void* front, void* dst, long long rows, int T, long long fe) {
    const size_t es = dtype_size(t);
    for (int j = 0; j < 2 && ok(); ++j) {
      char* d = (char*)dst + (size_t)j * fe * es;
      if (T - 2 + j >= 0) cuda(launch_copy_frames(t, (const char*)x + (size_t)(T - 2 + j) * fe * es, d, (int)rows, (long long)T * fe, 2 * fe, fe, s), "cache tail");
      else if (front) cuda(launch_copy_frames(t, (const char*)front + (size_t)(T + j) * fe * es, d, (int)rows, 2 * fe, 2 * fe, fe, s), "cache tail");
      else cuda(cudaMemset2DAsync(d, 2 * fe * es, 0, fe * es, (size_t)rows, s), "cache tail");
    }
  }
  // dst [rows][2 + T][fe] := [front (2 frames) | x (T frames)]
  void cat2(DType t, const void* front, const void* x, void* dst, long long rows, int T, long long fe) {
    const size_t es = dtype_size(t);
    cuda(launch_copy_frames(t, front, dst, (int)rows, 2 * fe, (2 + T) * fe, 2 * fe, s), "cache cat");
    cuda(launch_copy_frames(t, x, (char*)dst + 2 * fe * es, (int)rows, (long long)T * fe, (2 + T) * fe, (long long)T * fe, s), "cache cat");
  }
  // v1.0 stream, a conv whose input is the caller's fp32 NCDHW tensor (k = 3 in time): the cache holds the last two padded
  // input frames in that layout; later chunks run over [cache | chunk] and drop the two cached output frames, so the conv
  // kernel and its summation order are the whole clip's.
  Act conv_ext_stream(const ConvW& w, const float* x, int B, int C, int T, int H, int W, int t_rep, const std::string& key, ConvOpt o) {
    Act out;
    const long long rows = (long long)B * C, fe = (long long)H * W;
    CacheBuf* cb = cache(key, (size_t)rows * 2 * fe * sizeof(float));
    if (!cb) return out;
    Act in;
    in.B = B; in.C = C; in.H = H; in.W = W;
    if (ck->first) {
      in.p = (void*)x; in.T = T;
      o.ext_in = x; o.t_rep = t_rep;
      out = conv(w, in, o);
      if (ok() && !dry) {
        if (t_rep > 0 && T == 1) {   // padded input [x0 ... x0]
          for (int j = 0; j < 2; ++j)
            cuda(launch_copy_frames(DT_F32, x, (float*)cb->out() + j * fe, (int)rows, fe, 2 * fe, fe, s), "cache tail");
        } else {
          tail2(DT_F32, x, nullptr, cb->out(), rows, T, fe);
        }
      }
    } else {
      float* xc = (float*)alloc((size_t)rows * (2 + T) * fe * sizeof(float));
      if (!ok()) return out;
      if (!dry) {
        cat2(DT_F32, cb->in(), x, xc, rows, T, fe);
        tail2(DT_F32, x, cb->in(), cb->out(), rows, T, fe);
      }
      in.p = xc; in.T = 2 + T;
      o.ext_in = xc; o.to_off = 2;
      out = conv(w, in, o);
      ar.release(xc);
    }
    commit(cb);
    return out;
  }

  // ---- convolution ----------------------------------------------------------------------------
  // The descriptor conv(w, in, o) launches, but for the chunk-cache pointers: extents, strides, padding, time mode, residual.
  bool conv_desc(const ConvW& w, const Act& in, const ConvOpt& o, ConvP& p) {
    const bool v11 = m->desc.version == 1;
    p = conv_p(in.B, in.T, in.H, in.W, in.C);
    if (in.C != w.Ci) { rc = fail(VT_ERR_INVALID, "conv: Cin mismatch %d vs %d", in.C, w.Ci); return false; }
    if (o.ext_in && o.ext_in_indices) {
      Strides is = ncdhw_strides(1, in.T, in.H, in.W);   // the int32 token tensor [B,T,H,W]: no channel axis
      is.C = 0;
      set_in(p, is);
      p.fsq_d = m->desc.fsq_num_levels;
      for (int i = 0; i < VT_MAX_FSQ && i < p.fsq_d; ++i) p.fsq_levels[i] = m->desc.fsq_levels[i];
    } else if (o.ext_in) {
      set_in(p, ncdhw_strides(in.C, in.T, in.H, in.W));
    } else {
      // (stride overrides in ConvOpt count storage elements: bf16 values for split rows)
      set_in(p, cl_strides(in.T, in.H, in.W, in.C, cw, o.in_bs));
    }
    p.split = split ? 1 : 0;
    p.acc_scale = split ? 1.0f / w.wscale3 : 1.0f;
    p.kt = w.kt; p.kh = w.kh; p.kw = w.kw;
    p.st = o.st; p.sh = o.sh; p.sw = o.sw;
    p.ut = o.ut; p.uh = o.uh; p.uw = o.uw;
    p.t_rep = o.t_rep; p.to_off = o.to_off;
    // time padding: causal front pad (model_3dcausal.py:177), or -- non-causal family -- symmetric zero padding for stride 1
    // and one zero frame behind the end for the stride-2 time-downsample conv (model_3dnoncausal.py:80,86-87,101,203,271)
    int ptf = o.pt_front, ptb = o.pt_back;
    if (ptf < 0 && m->desc.noncausal && w.kt > 1) {
      if (o.st == 1) ptf = ptb = (w.kt - 1) / 2;
      else { ptf = 0; ptb = 1; }
    }
    p.pt = ptf >= 0 ? ptf : (w.kt - 1) + (1 - o.st);
    const int hp = (w.kh - 1) + (1 - o.sh), wp = (w.kw - 1) + (1 - o.sw);   // :178-179
    const int ph0 = o.ph0 >= 0 ? o.ph0 : hp / 2, ph1 = o.ph1 >= 0 ? o.ph1 : hp - hp / 2;
    const int pw0 = o.pw0 >= 0 ? o.pw0 : wp / 2, pw1 = o.pw1 >= 0 ? o.pw1 : wp - wp / 2;
    p.ph = ph0; p.pw = pw0;
    p.Co = w.Co;
    if (!conv_out_size(p, ptb, ph1, pw1)) { rc = fail(VT_ERR_INVALID, "conv: empty output"); return false; }
    if (o.ext_out) set_out(p, ncdhw_strides(p.Co, p.To, p.Ho, p.Wo));
    else if (o.out_view) set_out(p, Strides{o.ov_sB, o.ov_sT, o.ov_sH, o.ov_sW, 1});
    else set_out(p, cl_strides(p.To, p.Ho, p.Wo, p.Co, cw));
    // time padding mode: zeros, replicate (v1.1), or the chunk cache on a later chunk of a stream
    const bool cached = streaming() && o.cache_key && !ck->first;
    if (v11 && w.kt > 1) p.t_mode = 1;
    if (w.kt > 1 && cached) { p.t_mode = 2; p.cacheT = p.pt; }   // (folded 2x time upsampling: frames of the upsampled axis)
    p.bias = w.bias;
    p.res_mode = o.res_mode;
    p.ra = o.ra; p.rb = o.rb;
    if (o.res_mode) {
      const Act& r = *o.res;
      if (r.C != w.Co) { rc = fail(VT_ERR_INVALID, "conv: residual channel mismatch"); return false; }
      p.res = r.p;
      set_res(p, cl_strides(r.T, r.H, r.W, r.C, cw, o.res_bs));
      p.resT = r.T;
      if (o.res_mode == 3) {
        p.res_pool_off = o.res_pool_off;
        p.res_t_mode = cached ? 2 : (v11 ? 1 : 0);   // v1.1: replicate (model_3dcausal_v1_1.py:293-294)
      }
    }
    return true;
  }
  // The wgmma plan of conv(w, in, o) for its descriptor p, with the epilogues o requests; false: the conv does not run on conv_tc.
  bool tc_plan(const ConvW& w, const ConvP& p, const ConvOpt& o, TcPlan* pl) const {
    if (!tcm || o.force_simt || o.ext_in || !w.Kpad) return false;
    TcLnFusion lf;
    const NormW* ln = o.ln1 ? o.ln1 : o.ln2;
    if (ln && m->desc.norm_type == VT_NORM_LAYERNORM) {
      lf.mode = o.ln1 ? 1 : 2; lf.silu = o.ln1 ? o.ln1_silu : o.ln2_silu; lf.gamma = ln->gamma; lf.beta = ln->beta; lf.out2 = o.ln2_view;
    }
    return conv_tc_plan(p, o.ext_out ? DT_F32 : ta, &lf, o.reg, 1, pl);
  }
  // whether conv(w, in, o) would fuse LayerNorm ln (the next stage's norm) into its epilogue
  bool fuses_ln(const ConvW& w, const Act& in, ConvOpt o, const NormW* ln, bool silu) {
    o.ln2 = ln; o.ln2_silu = silu;
    ConvP p;
    TcPlan pl;
    return ln && conv_desc(w, in, o, p) && tc_plan(w, p, o, &pl) && pl.ln.mode != 0;
  }
  Act conv(const ConvW& w, const Act& in, const ConvOpt& o) {
    Act out;
    ConvP p;
    if (!ok() || !conv_desc(w, in, o, p)) return out;
    out.B = in.B; out.T = p.To; out.H = p.Ho; out.W = p.Wo; out.C = w.Co;
    out.p = o.ext_out ? (void*)o.ext_out : o.out_view;
    if (!out.p) { out.p = alloc((size_t)out.elems() * dtype_size(ta)); out.owned = true; }
    if (!ok()) return out;
    CacheBuf* cb = nullptr;
    int cache_off = 0;
    if (w.kt > 1 && streaming() && o.cache_key) {
      cache_off = cache_offset_for(o.cache_key);
      cb = cache(o.cache_key, (size_t)in.B * p.pt * in.frame() * dtype_size(o.ext_in ? DT_F32 : ta));
      if (!cb) return out;
      if (p.t_mode == 2) p.cache = cb->in();
    }
    CacheBuf* pc = nullptr;   // avg-pool branch of res_mode 3
    if (o.res_mode == 3 && streaming() && o.cache_key) {
      const Act& r = *o.res;
      pc = cache(std::string(o.cache_key) + "#pool", (size_t)r.B * r.frame() * dtype_size(ta));
      if (!pc) return out;
      if (p.res_t_mode == 2) p.res_cache = pc->in();
    }
    const DType tin = o.ext_in ? DT_F32 : ta;
    const DType tout = o.ext_out ? DT_F32 : ta;
    TcPlan pl;
    const bool tc = tc_plan(w, p, o, &pl);
    o.fused1 = tc && pl.ln.mode == 1;
    o.fused2 = tc && pl.ln.mode == 2;
    o.fused_reg = tc && pl.reg.mode != 0;
    if (o.fused2 && !o.out_view) {
      o.ln2_act = new_act(out.B, out.T, out.H, out.W, out.C);
      pl.ln.out2 = o.ln2_act.p;
      if (!ok()) return out;
    }
    if (!dry) {
      const bf16* wst = split ? w.w_stem3 : w.w_stem;
      const bool stem = tcm && !o.force_simt && o.ext_in && !o.ext_in_indices && !o.ext_out && !o.out_view && w.stem && conv_stem_supported(p);
      if (tc) {
        void* optr = (o.fused_reg && o.reg_only) ? nullptr : out.p;
        if (!cuda(launch_conv_tc(pl, (const bf16*)in.p, split ? w.w_nk3 : w.w_nk, optr, s), conv_tc_last_error())) return out;
      } else if (stem) {
        if (!cuda(launch_conv_stem(p, o.ext_in, wst, (bf16*)out.p, s), "conv_stem")) return out;
      } else if (!w.w_kn) {
        rc = fail(VT_ERR_INVALID, "phase-collapsed conv rejected by the wgmma path: %s", conv_tc_last_error());
        return out;
      } else {
        if (!cuda(launch_conv_simt(p, tin, tout, ta, o.ext_in ? (const void*)o.ext_in : in.p, w.w_kn, out.p, s), "conv_simt")) return out;
      }
      // cache := tail of the padded input (after the conv consumed the old cache)
      if (cb) {
        if (o.ut == 2) {
          // v1.0 folded 2x time upsampling: the last two upsampled frames are the last input frame twice
          const char* last = (const char*)in.p + (size_t)(in.T - 1) * in.frame() * dtype_size(tin);
          for (int j = 0; j < 2 && ok(); ++j)
            cuda(launch_copy_frames(tin, last, (char*)cb->out() + (size_t)j * in.frame() * dtype_size(tin), in.B, (long long)in.T * in.frame(),
                                    2 * in.frame(), in.frame(), s), "cache_update");
          if (!ok()) return out;
        } else {
          // v1.0: zero frames in front of the first chunk (v1.1 replicates frame 0)
          const bool zero_front = m->desc.version == 0 && ck->first;
          if (zero_front && !cuda(cudaMemsetAsync(cb->in(), 0, cb->bytes, s), "cache_update")) return out;
          if (!cuda(launch_cache_update(tin, o.ext_in ? (const void*)o.ext_in : in.p, cb->in(), cb->out(), in.B, in.T,
                                        p.pt, cache_off, ck->first && !zero_front, in.frame(), o.ext_in ? p.isB : p.isB / cw, s), "cache_update")) return out;
        }
        commit(cb);
      }
      if (pc) {
        // avg-pool branch cache = last frame of the padded input (model_3dcausal_v1_1.py:298)
        const Act& r = *o.res;
        if (!cuda(launch_copy_frames(ta, (const char*)r.p + (size_t)(r.T - 1) * r.frame() * dtype_size(ta), pc->out(), r.B,
                                     (long long)r.T * r.frame(), r.frame(), r.frame(), s), "pool cache")) return out;
        commit(pc);
      }
    }
    return out;
  }
  // ext_in path needs channels-last cache update from an NCDHW tensor: only conv_in of the encoder; handled by
  // converting the chunk to channels-last first (see run_encoder).

  Act norm(const NormW& n, const Act& in, bool silu, bool per_position) {
    Act out;
    if (!ok()) return out;
    out = new_act(in.B, in.T, in.H, in.W, in.C);
    if (!ok() || dry) {
      if (m->desc.norm_type == VT_NORM_GROUPNORM && !per_position && ok()) {
        void* st = alloc((size_t)in.B * in.T * 32 * 2 * sizeof(float));
        ar.release(st);
      }
      return out;
    }
    if (m->desc.norm_type == VT_NORM_LAYERNORM) {
      cuda(launch_layernorm(ta, in.p, n.gamma, n.beta, out.p, (long long)in.B * in.T * in.H * in.W, in.C, silu, exact, s), "layernorm");
    } else {
      float* st = nullptr;
      if (!per_position) st = (float*)alloc((size_t)in.B * in.T * 32 * 2 * sizeof(float));
      if (ok())
        cuda(launch_groupnorm(ta, in.p, n.gamma, n.beta, out.p, (long long)in.B * in.T, (long long)in.H * in.W, in.C,
                              per_position, silu, exact, st, s), "groupnorm");
      if (st) ar.release(st);
    }
    return out;
  }

  // The residual stream: x plus, when the producing conv's epilogue already made it, n = act(LN_{n_of}(x)).
  struct Stream {
    Act x, n;
    const NormW* n_of = nullptr;
  };
  Act take_norm(Stream& st, const NormW& nw, bool silu, bool per_position) {
    if (st.n.p && st.n_of == &nw) {
      Act r = st.n;
      st.n = Act();
      st.n_of = nullptr;
      return r;
    }
    return norm(nw, st.x, silu, per_position);
  }
  void set_stream(Stream& st, Act out, const ConvOpt& o) {
    if (st.n.p) free_act(st.n);
    free_act(st.x);
    st.x = out;
    st.n = Act();
    st.n_of = nullptr;
    if (o.fused2) { st.n = o.ln2_act; st.n_of = o.ln2; }
  }
  // ResnetBlock (2D, model_3dcausal.py:317-337), ResnetCausalBlock1D (:473-499; GroupNorm statistics per position, see
  // the oracle) and ResnetCausalBlock (3D, :400-424) share one shape: LN,SiLU,conv1,LN,SiLU,conv2,+skip.
  // `next`: the norm the FOLLOWING stage applies to this block's output (fused into conv2's epilogue when possible).
  // ResnetCausalBlock1D as ONE launch (tblock_tc.cu): BF16 mode, v1.0 zero padding, LayerNorm, 128 channels
  bool resblock1d_fused(const ResBlockW& r, Stream& st, const NormW* next, bool next_silu) {
    if (prec != VT_PREC_BF16 || m->desc.version != 0 || m->desc.noncausal || m->desc.norm_type != VT_NORM_LAYERNORM) return false;
    if (r.c1.Ci != 128 || r.c1.Co != 128 || r.c2.Co != 128 || r.c1.kt != 3 || r.c1.kh != 1) return false;
    if (!tblock_tc_supported(st.x.B, st.x.T, st.x.H, st.x.W, st.x.C)) return false;
    // streaming: the conv1 / conv2 caches of the two-launch path (n1 and LN2(h) frames t-2, t-1), read and written in-kernel
    CacheBuf* cc[2] = {nullptr, nullptr};
    TbCache tc;
    if (streaming()) {
      const size_t cbytes = (size_t)st.x.B * 2 * st.x.frame() * sizeof(bf16);
      cc[0] = cache(r.key + ".conv1", cbytes);
      if (cc[0]) cc[1] = cache(r.key + ".conv2", cbytes);
      if (!cc[1]) return true;
      if (!ck->first) { tc.n1_in = (const bf16*)cc[0]->in(); tc.h_in = (const bf16*)cc[1]->in(); }
      tc.n1_out = (bf16*)cc[0]->out(); tc.h_out = (bf16*)cc[1]->out();
    }
    Act n1 = take_norm(st, r.n1, true, true);
    Act out = new_act(st.x.B, st.x.T, st.x.H, st.x.W, 128);
    Act out2;
    if (next) out2 = new_act(st.x.B, st.x.T, st.x.H, st.x.W, 128);
    if (ok() && !dry) {
      cuda(launch_tblock_tc((const bf16*)n1.p, (const bf16*)st.x.p, r.c1.w_nk, r.c1.bias, r.n2.gamma, r.n2.beta, r.c2.w_nk, r.c2.bias,
                            (bf16*)out.p, next ? (bf16*)out2.p : nullptr, next ? next->gamma : nullptr, next ? next->beta : nullptr,
                            next_silu, st.x.B, st.x.T, st.x.H, st.x.W, s, cc[0] ? &tc : nullptr), tblock_tc_last_error());
      commit(cc[0]);
      commit(cc[1]);
    }
    free_act(n1);
    if (st.n.p) free_act(st.n);
    free_act(st.x);
    st.x = out;
    st.n = out2;
    st.n_of = next ? next : nullptr;
    return true;
  }
  void resblock(const ResBlockW& r, Stream& st, int kind /*2,1,3*/, const NormW* next, bool next_silu) {
    const bool pp = kind == 1;
    if (kind == 1 && resblock1d_fused(r, st, next, next_silu)) return;
    const std::string k1 = r.key + ".conv1", k2 = r.key + ".conv2";
    Act n1 = take_norm(st, r.n1, true, pp);
    ConvOpt o1;
    if (kind != 2) o1.cache_key = k1.c_str();
    o1.ln1 = &r.n2;
    Act h1 = conv(r.c1, n1, o1);
    free_act(n1);
    Act n2 = h1;
    if (!o1.fused1) {
      n2 = norm(r.n2, h1, true, pp);
      free_act(h1);
    }
    Act skip = st.x;
    if (r.has_nin) skip = conv(r.nin, st.x, ConvOpt());
    ConvOpt o;
    o.res_mode = 1; o.res = &skip;
    if (kind != 2) o.cache_key = k2.c_str();
    o.ln2 = next; o.ln2_silu = next_silu;
    Act out = conv(r.c2, n2, o);
    free_act(n2);
    if (r.has_nin) free_act(skip);
    set_stream(st, out, o);
  }
  // wgmma path of the attention core: S = scale * Q K^T (fp32), P = softmax(S) (bf16), O = P V.
  // Both products are the conv_tc GEMM with per-frame "weights": K of the frame for the scores, V^T for the output.
  bool attention_tc(const Act& q, const Act& k, const Act& v, Act& o) {
    const int frames = q.B * q.T, tokens = q.H * q.W, C = q.C;
    if (!tcm || tokens % 64 != 0 || C % 64 != 0 || tokens % 32 != 0) return false;
    ConvP ps = conv_p(frames, 1, q.H, q.W, C);
    ps.split = split ? 1 : 0;
    set_in(ps, cl_strides(1, q.H, q.W, C, cw));
    ps.To = 1; ps.Ho = q.H; ps.Wo = q.W; ps.Co = tokens;
    set_out(ps, cl_strides(1, q.H, q.W, tokens, 1));   // fp32 scores
    ps.kt = ps.kh = ps.kw = 1;
    ps.ra = 0.f; ps.rb = 1.0f / sqrtf((float)C);
    ConvP pv = ps;
    pv.Ci = tokens; set_in(pv, cl_strides(1, q.H, q.W, tokens, cw));
    pv.Co = C; set_out(pv, cl_strides(1, q.H, q.W, C, cw));
    pv.rb = 1.0f;
    TcPlan pls, plv;
    if (!conv_tc_plan(ps, DT_F32, nullptr, nullptr, frames, &pls) || !conv_tc_plan(pv, ta, nullptr, nullptr, frames, &plv)) return false;
    o = new_act(q.B, q.T, q.H, q.W, C);
    float* S = (float*)alloc((size_t)frames * tokens * tokens * sizeof(float));
    bf16* P = (bf16*)alloc((size_t)frames * tokens * tokens * dtype_size(ta));
    bf16* Vt = (bf16*)alloc((size_t)frames * tokens * C * dtype_size(ta));
    if (ok() && !dry) {
      // per-frame "weights": K of the frame ([tokens][C], split: [tokens][hi C | lo C]) and V^T ([C][tokens])
      cuda(launch_conv_tc(pls, (const bf16*)q.p, (const bf16*)k.p, S, s, (long long)tokens * C * cw), conv_tc_last_error());
      cuda(launch_softmax_rows(ta, S, P, (long long)frames * tokens, tokens, s), "attn softmax");
      cuda(launch_transpose_bf16((const bf16*)v.p, Vt, frames, tokens, C, s, split), "attn transpose V");
      cuda(launch_conv_tc(plv, P, Vt, o.p, s, (long long)tokens * C * cw), conv_tc_last_error());
    }
    ar.release(Vt);
    ar.release(P);
    ar.release(S);
    return true;
  }
  // Frames above 32 x 32 positions: the fused kernel (attn_tc.cu), online softmax, no tokens x tokens buffer; its only
  // workspace is V^T, the size of v.  The choice depends on the frame (H, W, C) only, never on the frame count.  Frames of
  // up to 1024 tokens keep the two-GEMM path above, whose launch plans the production-plan table pins.
  bool attention_fused(const Act& q, const Act& k, const Act& v, Act& o) {
    const long long frames = (long long)q.B * q.T, tokens = (long long)q.H * q.W;
    if (!tcm || tokens <= 1024 || !attn_tc_supported(frames, tokens, q.C, split)) return false;
    o = new_act(q.B, q.T, q.H, q.W, q.C);
    void* vt = alloc(attn_tc_workspace(frames, tokens, q.C, split));
    if (ok() && !dry)
      cuda(launch_attn_tc((const bf16*)q.p, (const bf16*)k.p, (const bf16*)v.p, (bf16*)o.p, (int)frames, q.H, q.W, q.C, split, vt, s),
           attn_tc_last_error());
    ar.release(vt);
    return true;
  }
  Act attention_core(const Act& q, const Act& k, const Act& v) {
    const int frames = q.B * q.T, tokens = q.H * q.W, C = q.C;
    {
      Act o_tc;
      if (attention_fused(q, k, v, o_tc)) return o_tc;
      if (attention_tc(q, k, v, o_tc)) return o_tc;
    }
    Act o = new_act(q.B, q.T, q.H, q.W, C);
    if (split) {
      // shapes the wgmma path does not take (tiny test models): join hi|lo to fp32, fp32 FMA GEMMs, split the result
      const size_t nqc = (size_t)frames * tokens * C;
      float* S = (float*)alloc((size_t)frames * tokens * tokens * sizeof(float));
      float* P = (float*)alloc((size_t)frames * tokens * tokens * sizeof(float));
      float* qf = (float*)alloc(nqc * sizeof(float));
      float* kf = (float*)alloc(nqc * sizeof(float));
      float* vf = (float*)alloc(nqc * sizeof(float));
      float* of = (float*)alloc(nqc * sizeof(float));
      if (ok() && !dry) {
        const float scale = 1.0f / sqrtf((float)C);
        const long long qs = (long long)tokens * C, ss = (long long)tokens * tokens, rows = (long long)frames * tokens;
        cuda(launch_split_to_f32((const bf16*)q.p, qf, rows, C, s), "attn join q");
        cuda(launch_split_to_f32((const bf16*)k.p, kf, rows, C, s), "attn join k");
        cuda(launch_split_to_f32((const bf16*)v.p, vf, rows, C, s), "attn join v");
        cuda(launch_gemm_simt(DT_F32, DT_F32, DT_F32, qf, kf, S, tokens, tokens, C, C, C, 1, tokens, frames, qs, qs, ss, scale, s), "attn QK^T");
        cuda(launch_softmax_rows(DT_F32, S, P, rows, tokens, s), "attn softmax");
        cuda(launch_gemm_simt(DT_F32, DT_F32, DT_F32, P, vf, of, tokens, C, tokens, tokens, 1, C, C, frames, ss, qs, qs, 1.0f, s), "attn PV");
        cuda(launch_f32_to_split(of, (bf16*)o.p, rows, C, s), "attn split o");
      }
      ar.release(of); ar.release(vf); ar.release(kf); ar.release(qf); ar.release(P); ar.release(S);
      return o;
    }
    float* S = (float*)alloc((size_t)frames * tokens * tokens * sizeof(float));
    void* P = alloc((size_t)frames * tokens * tokens * dtype_size(ta));
    if (ok() && !dry) {
      const float scale = 1.0f / sqrtf((float)C);
      const long long qs = (long long)tokens * C, ss = (long long)tokens * tokens;
      cuda(launch_gemm_simt(ta, ta, DT_F32, q.p, k.p, S, tokens, tokens, C, C, C, 1, tokens, frames, qs, qs, ss, scale, s), "attn QK^T");
      cuda(launch_softmax_rows(ta, S, P, (long long)frames * tokens, tokens, s), "attn softmax");
      cuda(launch_gemm_simt(ta, ta, ta, P, v.p, o.p, tokens, C, tokens, tokens, 1, C, C, frames, ss, qs, qs, 1.0f, s), "attn PV");
    }
    ar.release(P);
    ar.release(S);
    return o;
  }
  // AttnBlockWrapper: model_3dcausal.py:114-141
  void attn(const AttnW& a, Stream& st, const NormW* next, bool next_silu) {
    Act n = take_norm(st, a.n, false, false);
    Act q = conv(a.q, n, ConvOpt());
    Act k = conv(a.k, n, ConvOpt());
    Act v = conv(a.v, n, ConvOpt());
    free_act(n);
    Act o = attention_core(q, k, v);
    free_act(q); free_act(k); free_act(v);
    ConvOpt op; op.res_mode = 1; op.res = &st.x;
    op.ln2 = next; op.ln2_silu = next_silu;
    Act out = conv(a.proj, o, op);
    free_act(o);
    set_stream(st, out, op);
  }
  Act upsample_mat(const Act& x, int ut, int uh, int uw) {
    Act y = new_act(x.B, x.T * ut, x.H * uh, x.W * uw, x.C);
    if (ok() && !dry) cuda(launch_upsample_nearest(ta, x.p, y.p, x.B, x.T, x.H, x.W, x.C, ut, uh, uw, s), "upsample_nearest");
    return y;
  }
  bool fold_upsample() const { return prec == VT_PREC_FMA32; }

  // Downsample: pad (0,1,0,1) + conv3x3 stride 2 (model_3dcausal.py:223-227)
  void down(const LevelW& lv, Stream& st, const NormW* next, bool next_silu) {
    ConvOpt o; o.sh = 2; o.sw = 2; o.ph0 = 0; o.ph1 = 1; o.pw0 = 0; o.pw1 = 1;
    o.ln2 = next; o.ln2_silu = next_silu;
    Act y = conv(lv.resample, st.x, o);
    set_stream(st, y, o);
  }
  // TimeDownsampleResCausal2x: model_3dcausal.py:247-252 / model_3dcausal_v1_1.py:289-302
  void time_down(const LevelW& lv, Stream& st, const NormW* next, bool next_silu) {
    const std::string ck_ = lv.tkey + ".conv";
    ConvOpt o;
    o.st = 2; o.res_mode = 3; o.res = &st.x; o.ra = lv.alpha; o.rb = 1.f - lv.alpha; o.cache_key = ck_.c_str();
    if (m->desc.noncausal) o.res_pool_off = 1;   // avg-pool window 2t .. 2t+2, zero frame behind the end (model_3dnoncausal.py:86-88)
    o.ln2 = next; o.ln2_silu = next_silu;
    Act out = conv(lv.tconv, st.x, o);
    set_stream(st, out, o);
  }
  // Upsample: nearest 2x (H,W) + conv3x3 (model_3dcausal.py:208-212)
  void up(const LevelW& lv, Stream& st, const NormW* next, bool next_silu) {
    Act& h = st.x;
    if (fold_upsample()) {
      ConvOpt o; o.uh = 2; o.uw = 2;
      Act y = conv(lv.resample, h, o);
      set_stream(st, y, o);
    } else if (lv.has_up_phase && tcm) {
      // four parity classes of the 2x-upsampled output, each a 1x2x2 conv on the low-resolution input
      Act y = new_act(h.B, h.T, 2 * h.H, 2 * h.W, lv.resample.Co);
      const long long C = lv.resample.Co, Wo2 = 2 * h.W, Ho2 = 2 * h.H;
      auto phase = [&](int py, int px, const Act* n) {   // n: where the fused LayerNorm of the next stage goes
        ConvOpt o;
        o.ph0 = py == 0 ? 1 : 0; o.ph1 = 1 - o.ph0; o.pw0 = px == 0 ? 1 : 0; o.pw1 = 1 - o.pw0;
        const size_t off = (size_t)((py * Wo2 + px) * C) * dtype_size(ta);
        o.out_view = dry ? y.p : (void*)((char*)y.p + off);
        o.ov_sW = 2 * C * cw; o.ov_sH = 2 * Wo2 * C * cw; o.ov_sT = Ho2 * Wo2 * C * cw; o.ov_sB = o.ov_sT * h.T;
        if (n) { o.ln2 = next; o.ln2_silu = next_silu; o.ln2_view = dry ? n->p : (void*)((char*)n->p + off); }
        return o;
      };
      // the next stage's LayerNorm is fused when the first phase conv's plan takes it (else that stage normalises)
      const bool fuse = fuses_ln(lv.up_ph[0], h, phase(0, 0, nullptr), next, next_silu);
      Act n;
      if (fuse) n = new_act(h.B, h.T, 2 * h.H, 2 * h.W, lv.resample.Co);
      for (int py = 0; py < 2 && ok(); ++py)
        for (int px = 0; px < 2 && ok(); ++px) {
          ConvOpt o = phase(py, px, fuse ? &n : nullptr);
          conv(lv.up_ph[py * 2 + px], h, o);
          if (fuse && ok() && !o.fused2) rc = fail(VT_ERR_INVALID, "upsample phase conv did not fuse its LayerNorm");
        }
      set_stream(st, y, ConvOpt());
      if (fuse) { st.n = n; st.n_of = next; }
    } else {
      Act hu = upsample_mat(h, 1, 2, 2);
      ConvOpt o; o.ln2 = next; o.ln2_silu = next_silu;
      Act y = conv(lv.resample, hu, o);
      free_act(hu);
      set_stream(st, y, o);
    }
  }
  // TimeUpsampleResCausal2x: model_3dcausal.py:267-273 / model_3dcausal_v1_1.py:325-343
  void time_up(const LevelW& lv, Stream& st, const NormW* next, bool next_silu) {
    Act x = st.x;          // consumed here; st.x is re-pointed by set_stream at every exit
    st.x = Act();
    const bool v11 = m->desc.version == 1;
    const std::string ckey = lv.tkey + ".conv";
    ConvOpt o;
    o.ra = lv.alpha; o.rb = 1.f - lv.alpha; o.cache_key = ckey.c_str();
    o.ln2 = next; o.ln2_silu = next_silu;
    if (!v11) {
      if (fold_upsample()) {
        o.ut = 2; o.res_mode = 2; o.res = &x;
        Act out = conv(lv.tconv, x, o);
        free_act(x);
        set_stream(st, out, o);
        return;
      }
      if (lv.has_tup_phase && tcm) {
        // even / odd output frames: 2x3x3 convs on the un-upsampled input, mixed with x[t/2] in the epilogue
        Act out = new_act(x.B, 2 * x.T, x.H, x.W, lv.tconv.Co);
        const long long fr = (long long)x.H * x.W * lv.tconv.Co;
        const std::string pk[2] = {ckey + "#ph0", ckey + "#ph1"};   // streaming: each parity keeps its own copy of x[-1]
        auto phase = [&](int pt, const Act* n) {   // n: where the fused LayerNorm of the next stage goes
          ConvOpt op;
          op.ra = lv.alpha; op.rb = 1.f - lv.alpha; op.res_mode = 1; op.res = &x;
          if (m->desc.noncausal) { op.pt_front = pt == 0 ? 1 : 0; op.pt_back = pt == 0 ? 0 : 1; }   // frames (i-1, i) / (i, i+1)
          op.cache_key = pk[pt].c_str();
          const size_t off = (size_t)(pt * fr) * dtype_size(ta);
          op.out_view = dry ? out.p : (void*)((char*)out.p + off);
          op.ov_sW = (long long)lv.tconv.Co * cw; op.ov_sH = (long long)x.W * lv.tconv.Co * cw; op.ov_sT = 2 * fr * cw; op.ov_sB = 2 * fr * x.T * cw;
          if (n) { op.ln2 = next; op.ln2_silu = next_silu; op.ln2_view = dry ? n->p : (void*)((char*)n->p + off); }
          return op;
        };
        const bool fuse = fuses_ln(lv.tup_ph[0], x, phase(0, nullptr), next, next_silu);
        Act n;
        if (fuse) n = new_act(x.B, 2 * x.T, x.H, x.W, lv.tconv.Co);
        for (int pt = 0; pt < 2 && ok(); ++pt) {
          ConvOpt op = phase(pt, fuse ? &n : nullptr);
          conv(lv.tup_ph[pt], x, op);
          if (fuse && ok() && !op.fused2) rc = fail(VT_ERR_INVALID, "time-upsample phase conv did not fuse its LayerNorm");
        }
        free_act(x);
        set_stream(st, out, ConvOpt());
        if (fuse) { st.n = n; st.n_of = next; }
        return;
      }
      Act xu = upsample_mat(x, 2, 1, 1);
      free_act(x);
      o.res_mode = 1; o.res = &xu;
      Act out = conv(lv.tconv, xu, o);
      free_act(xu);
      set_stream(st, out, o);
      return;
    }
    if (m->desc.interpolation_mode != VT_INTERP_TRILINEAR) {
      Act xu = upsample_mat(x, 2, 1, 1);
      free_act(x);
      o.res_mode = 1; o.res = &xu;
      Act out = conv(lv.tconv, xu, o);
      free_act(xu);
      set_stream(st, out, o);
      return;
    }
    // trilinear with cache (model_3dcausal_v1_1.py:329-340)
    const int n = lv.num_temp_upsample;
    const long long fe = x.frame();
    const size_t es = dtype_size(ta);
    const bool persist = ck && ck->persist;
    const bool first = !ck || ck->first;
    CacheBuf* cb = nullptr;
    if (persist) {
      cb = cache(lv.tkey + "#up", (size_t)x.B * n * fe * es);
      if (!cb) { free_act(x); return; }
    }
    Act xu;
    Act view;
    long long bs = -1;
    Act big;  // storage that backs `view` when it is a sub-range
    if (first) {
      // x[:n] and x[n:] interpolated separately, concatenated
      xu = new_act(x.B, 2 * x.T, x.H, x.W, x.C);
      if (ok() && !dry) {
        const int na = std::min(n, x.T), nb = x.T - na;
        // part a: frames [0,na) -> out frames [0,2na); part b: frames [na,T) -> out frames [2na,2T)
        // both read/write with batch strides of the full tensors: run per part through strided views
        for (int b = 0; b < x.B && ok(); ++b) {
          const char* xb = (const char*)x.p + (size_t)b * x.T * fe * es;
          char* yb = (char*)xu.p + (size_t)b * 2 * x.T * fe * es;
          cuda(launch_time_interp2x(ta, xb, yb, 1, na, (long long)x.H * x.W, x.C, s), "time_interp2x");
          if (nb > 0) cuda(launch_time_interp2x(ta, xb + (size_t)na * fe * es, yb + (size_t)2 * na * fe * es, 1, nb, (long long)x.H * x.W, x.C, s), "time_interp2x");
        }
        if (cb) {  // cache = x[:, -n:]
          if (x.T < n) { rc = fail(VT_ERR_INVALID, "time_up: first chunk shorter than num_temp_upsample"); }
          else cuda(launch_copy_frames(ta, (const char*)x.p + (size_t)(x.T - n) * fe * es, cb->out(), x.B, (long long)x.T * fe, (long long)n * fe, (long long)n * fe, s), "up cache");
          commit(cb);
        }
      }
      view = xu;
    } else {
      // xc = cat(cache, x); cache = xc[-2n:-n]; x' = interp(xc)[2n:]
      Act xc = new_act(x.B, n + x.T, x.H, x.W, x.C);
      big = new_act(x.B, 2 * (n + x.T), x.H, x.W, x.C);
      if (ok() && !dry) {
        cuda(launch_copy_frames(ta, cb->in(), xc.p, x.B, (long long)n * fe, (long long)(n + x.T) * fe, (long long)n * fe, s), "up cat a");
        cuda(launch_copy_frames(ta, x.p, (char*)xc.p + (size_t)n * fe * es, x.B, (long long)x.T * fe, (long long)(n + x.T) * fe, (long long)x.T * fe, s), "up cat b");
        cuda(launch_copy_frames(ta, (const char*)xc.p + (size_t)(x.T - n) * fe * es, cb->out(), x.B, (long long)(n + x.T) * fe, (long long)n * fe, (long long)n * fe, s), "up cache");
        commit(cb);
        cuda(launch_time_interp2x(ta, xc.p, big.p, x.B, n + x.T, (long long)x.H * x.W, x.C, s), "time_interp2x");
      }
      free_act(xc);
      view = big;
      view.owned = false;
      view.p = (char*)big.p + (size_t)2 * n * fe * es;
      view.T = 2 * x.T;
      bs = (long long)2 * (n + x.T) * fe * cw;
    }
    free_act(x);
    o.res_mode = 1; o.res = &view; o.in_bs = bs; o.res_bs = bs;
    Act out = conv(lv.tconv, view, o);
    if (first) free_act(xu); else free_act(big);
    set_stream(st, out, o);
  }
};

// ---- encoder / decoder stacks ----------------------------------------------------------------------
// The stack is flattened into stages so that each stream-producing conv knows which norm the NEXT stage applies to its
// output (and can fuse it into its epilogue).
struct Stage {
  enum Kind { RES2D, RES1D, RES3D, ATTN, DOWN, TDOWN, UP, TUP, HEAD } kind;
  const ResBlockW* rb = nullptr;
  const AttnW* at = nullptr;
  const LevelW* lv = nullptr;
  const NormW* head_norm = nullptr;
  const NormW* first_norm(bool* silu) const {
    *silu = true;
    switch (kind) {
      case RES2D: case RES1D: case RES3D: return &rb->n1;
      case ATTN: *silu = false; return &at->n;
      case HEAD: return head_norm;
      default: return nullptr;
    }
  }
};

static void run_stages(Exec& ex, Exec::Stream& st, const std::vector<Stage>& stages) {
  for (size_t i = 0; i < stages.size() && ex.ok(); ++i) {
    const Stage& sg = stages[i];
    bool nsilu = true;
    const NormW* next = (i + 1 < stages.size()) ? stages[i + 1].first_norm(&nsilu) : nullptr;
    switch (sg.kind) {
      case Stage::RES2D: ex.resblock(*sg.rb, st, 2, next, nsilu); break;
      case Stage::RES1D: ex.resblock(*sg.rb, st, 1, next, nsilu); break;
      case Stage::RES3D: ex.resblock(*sg.rb, st, 3, next, nsilu); break;
      case Stage::ATTN: ex.attn(*sg.at, st, next, nsilu); break;
      case Stage::DOWN: ex.down(*sg.lv, st, next, nsilu); break;
      case Stage::TDOWN: ex.time_down(*sg.lv, st, next, nsilu); break;
      case Stage::UP: ex.up(*sg.lv, st, next, nsilu); break;
      case Stage::TUP: ex.time_up(*sg.lv, st, next, nsilu); break;
      case Stage::HEAD: break;
    }
  }
}

// x_ext: fp32 [B,Cin,T,H,W]; h_out: fp32 [B,Cz,Tz,Hz,Wz].  reg (optional): regularizer outputs; when conv_out runs on the
// wgmma path it is applied in that kernel's epilogue (reg_done = true) and h_out is only written if want_h.
static void run_encoder(Exec& ex, const float* x_ext, int B, int T, int H, int W, float* h_out, const TcRegFusion* reg = nullptr,
                        bool want_h = true, bool* reg_done = nullptr) {
  if (reg_done) *reg_done = false;
  vt_model* m = ex.m;
  const vt_model_desc& d = m->desc;
  const StackW& e = m->enc;
  const int tdf = d.time_downsample_factor;
  int t_rep = 0;
  if (T % tdf != 0 && !d.noncausal) t_rep = (d.version == 0) ? (tdf - 1) : (tdf - T % tdf);  // model_3dcausal.py:685-689 / _v1_1.py:755-760
  Act xin;
  xin.p = (void*)x_ext; xin.B = B; xin.T = T; xin.H = H; xin.W = W; xin.C = d.in_channels;
  Exec::Stream st;
  if (ex.streaming() && ex.tcm && e.conv_in.stem && T + t_rep >= 2) {
    // chunked v1.1 / streamed v1.0 on the stem kernel: the causal cache (last two padded input frames,
    // model_3dcausal_v1_1.py:230-233) is kept in the caller's layout (fp32 [B,C,2,H,W]) and read by the kernel's patch loader
    CacheBuf* cb = ex.cache("encoder.conv_in#stem", (size_t)B * d.in_channels * 2 * H * W * sizeof(float));
    if (!cb) return;
    st.x = ex.new_act(B, T + t_rep, H, W, e.conv_in.Co);
    if (ex.ok() && !ex.dry) {
      ConvP p = stem_p(B, d.in_channels, T, H, W, e.conv_in.Co, t_rep, ex.split, e.conv_in.bias);
      p.acc_scale = ex.split ? 1.0f / e.conv_in.wscale3 : 1.0f;
      p.t_mode = ex.ck->first ? (d.version == 1 ? 1 : 0) : 2;   // first chunk: replicate (v1.1) / zero (v1.0) padding
      p.cache = cb->in(); p.cacheT = 2;
      if (!conv_stem_supported(p)) { ex.rc = fail(VT_ERR_INVALID, "stem kernel rejected the chunk geometry"); return; }
      ex.cuda(launch_conv_stem(p, x_ext, ex.split ? e.conv_in.w_stem3 : e.conv_in.w_stem, (bf16*)st.x.p, ex.s), "conv_stem");
      ex.cuda(launch_stem_cache_update(x_ext, (float*)cb->out(), B, d.in_channels, T, t_rep, H, W, ex.s), "stem cache");
      ex.commit(cb);
    }
  } else if (d.version == 1 && ex.ck && ex.ck->persist) {
    // chunked v1.1: the causal cache of conv_in holds *padded input* frames; materialise the replicate-padded chunk
    // channels-last so the cache update sees the same tensor the reference caches (model_3dcausal_v1_1.py:230-233).
    Act xp = ex.new_act(B, T + t_rep, H, W, d.in_channels);
    if (ex.ok() && !ex.dry) ex.cuda(launch_ncdhw_to_cl(ex.ta, x_ext, xp.p, B, d.in_channels, T, H, W, t_rep, ex.s), "ncdhw_to_cl");
    ConvOpt o; o.cache_key = "encoder.conv_in";
    st.x = ex.conv(e.conv_in, xp, o);
    ex.free_act(xp);
  } else if (ex.streaming()) {
    st.x = ex.conv_ext_stream(e.conv_in, x_ext, B, d.in_channels, T, H, W, t_rep, "encoder.conv_in", ConvOpt());
  } else {
    ConvOpt o; o.ext_in = x_ext; o.t_rep = t_rep;
    st.x = ex.conv(e.conv_in, xin, o);
  }
  std::vector<Stage> stages;
  for (size_t l = 0; l < e.levels.size(); ++l) {
    const LevelW& lv = e.levels[l];
    for (size_t b = 0; b < lv.blk.size(); ++b) {
      Stage a; a.kind = Stage::RES2D; a.rb = &lv.blk[b]; stages.push_back(a);
      Stage t; t.kind = Stage::RES1D; t.rb = &lv.tblk[b]; stages.push_back(t);
    }
    if (lv.has_resample) {
      Stage a; a.kind = Stage::DOWN; a.lv = &lv; stages.push_back(a);
      if (lv.has_tres) { Stage t; t.kind = Stage::TDOWN; t.lv = &lv; stages.push_back(t); }
    }
  }
  { Stage a; a.kind = Stage::RES3D; a.rb = &e.mid1; stages.push_back(a); }
  { Stage a; a.kind = Stage::ATTN; a.at = &e.attn; stages.push_back(a); }
  { Stage a; a.kind = Stage::RES3D; a.rb = &e.mid2; stages.push_back(a); }
  { Stage a; a.kind = Stage::HEAD; a.head_norm = &e.norm_out; stages.push_back(a); }
  run_stages(ex, st, stages);
  Act n = ex.take_norm(st, e.norm_out, true, false);
  ex.free_act(st.x);
  ConvOpt o; o.ext_out = h_out; o.cache_key = "encoder.conv_out";
  o.reg = reg; o.reg_only = !want_h;
  ex.conv(e.conv_out, n, o);
  if (reg_done) *reg_done = o.fused_reg;
  ex.free_act(n);
}

// z_ext: fp32 [B,z,Tz,Hz,Wz]; x_out: fp32 [B,out_ch,Tout,H,W]
static void run_decoder(Exec& ex, const float* z_ext, int B, int Tz, int Hz, int Wz, float* x_out, bool z_is_indices = false) {
  vt_model* m = ex.m;
  const vt_model_desc& d = m->desc;
  const StackW& g = m->dec;
  Act zin;
  zin.p = (void*)z_ext; zin.B = B; zin.T = Tz; zin.H = Hz; zin.W = Wz; zin.C = d.z_channels;
  Exec::Stream st;
  if (d.version == 1 && ex.ck && ex.ck->persist) {
    Act zp = ex.new_act(B, Tz, Hz, Wz, d.z_channels);
    if (ex.ok() && !ex.dry) ex.cuda(launch_ncdhw_to_cl(ex.ta, z_ext, zp.p, B, d.z_channels, Tz, Hz, Wz, 0, ex.s), "ncdhw_to_cl");
    ConvOpt o; o.cache_key = "decoder.conv_in";
    st.x = ex.conv(g.conv_in, zp, o);
    ex.free_act(zp);
  } else if (ex.streaming()) {
    if (z_is_indices) { ex.rc = fail(VT_ERR_INVALID, "a decoder stream takes latents, not token indices"); return; }
    st.x = ex.conv_ext_stream(g.conv_in, z_ext, B, d.z_channels, Tz, Hz, Wz, 0, "decoder.conv_in", ConvOpt());
  } else {
    ConvOpt o; o.ext_in = z_ext; o.ext_in_indices = z_is_indices;
    st.x = ex.conv(g.conv_in, zin, o);
  }
  std::vector<Stage> stages;
  { Stage a; a.kind = Stage::RES3D; a.rb = &g.mid1; stages.push_back(a); }
  { Stage a; a.kind = Stage::ATTN; a.at = &g.attn; stages.push_back(a); }
  { Stage a; a.kind = Stage::RES3D; a.rb = &g.mid2; stages.push_back(a); }
  for (int l = (int)g.levels.size() - 1; l >= 0; --l) {
    const LevelW& lv = g.levels[l];
    for (size_t b = 0; b < lv.blk.size(); ++b) {
      Stage a; a.kind = Stage::RES2D; a.rb = &lv.blk[b]; stages.push_back(a);
      Stage t; t.kind = Stage::RES1D; t.rb = &lv.tblk[b]; stages.push_back(t);
    }
    if (lv.has_resample) {
      Stage a; a.kind = Stage::UP; a.lv = &lv; stages.push_back(a);
      if (lv.has_tres) { Stage t; t.kind = Stage::TUP; t.lv = &lv; stages.push_back(t); }  // nested as model_3dcausal.py:844-853
    }
  }
  { Stage a; a.kind = Stage::HEAD; a.head_norm = &g.norm_out; stages.push_back(a); }
  run_stages(ex, st, stages);
  Act n = ex.take_norm(st, g.norm_out, true, false);
  ex.free_act(st.x);
  if (ex.prec == VT_PREC_BF16 && m->head_planes.Kpad > 0 && n.W % 8 == 0) {
    // 27 x 4 per-tap partial outputs by one GEMM over the input, then a gather-add of the shifted partials
    Act P = ex.conv(m->head_planes, n, ConvOpt());
    ex.free_act(n);
    if (ex.ok() && ex.streaming()) {
      // streamed v1.0: the cache holds the planes of the last two input frames; later chunks gather over [cache | planes]
      const long long fe = (long long)P.H * P.W * 128;
      CacheBuf* cb = ex.cache("decoder.conv_out#planes", (size_t)P.B * 2 * fe * sizeof(bf16));
      if (!cb) return;
      if (ex.ck->first) {
        if (!ex.dry) {
          ex.cuda(launch_tap_planes_gather((const bf16*)P.p, g.conv_out.bias, x_out, P.B, P.T, P.H, P.W, 128, g.conv_out.Co,
                                           d.time_downsample_factor - 1, ex.s), "tap_planes_gather");
          ex.tail2(DT_BF16, P.p, nullptr, cb->out(), P.B, P.T, fe);
        }
      } else {
        bf16* Pc = (bf16*)ex.alloc((size_t)P.B * (2 + P.T) * fe * sizeof(bf16));
        if (ex.ok() && !ex.dry) {
          ex.cat2(DT_BF16, cb->in(), P.p, Pc, P.B, P.T, fe);
          ex.tail2(DT_BF16, P.p, cb->in(), cb->out(), P.B, P.T, fe);
          ex.cuda(launch_tap_planes_gather(Pc, g.conv_out.bias, x_out, P.B, 2 + P.T, P.H, P.W, 128, g.conv_out.Co, 2, ex.s), "tap_planes_gather");
        }
        ex.ar.release(Pc);
      }
      ex.commit(cb);
    } else if (ex.ok() && !ex.dry) {
      ex.cuda(launch_tap_planes_gather((const bf16*)P.p, g.conv_out.bias, x_out, P.B, P.T, P.H, P.W, 128, g.conv_out.Co,
                                       d.noncausal ? 0 : d.time_downsample_factor - 1, ex.s, d.noncausal ? 1 : 2), "tap_planes_gather");
    }
    ex.free_act(P);
    return;
  }
  ConvOpt o; o.ext_out = x_out; o.cache_key = "decoder.conv_out";
  // model_3dcausal.py:883-885 (a stream drops the frames once, in its first chunk)
  if (d.version == 0 && !d.noncausal && (!ex.streaming() || ex.ck->first)) o.to_off = d.time_downsample_factor - 1;
  ex.conv(g.conv_out, n, o);
  ex.free_act(n);
}

static int latent_shape(const vt_model* m, int T, int H, int W, int* Tz, int* Hz, int* Wz) {
  const vt_model_desc& d = m->desc;
  const int tdf = d.time_downsample_factor;
  int t = T;
  if (T % tdf != 0 && !d.noncausal) t += (d.version == 0) ? (tdf - 1) : (tdf - T % tdf);
  int h = H, w = W;
  for (int l = 0; l < d.num_levels; ++l) {
    if (contains(m->spatial_ds, l)) {
      h = (h + 1 - 3) / 2 + 1;
      w = (w + 1 - 3) / 2 + 1;
      if (contains(m->tempo_ds, l)) t = (t + 1 - 3) / 2 + 1;
    }
  }
  *Tz = t; *Hz = h; *Wz = w;
  return VT_OK;
}
static void decoded_shape(const vt_model* m, int Tz, int Hz, int Wz, int* T, int* H, int* W) {
  const vt_model_desc& d = m->desc;
  int t = Tz, h = Hz, w = Wz;
  for (int l = d.num_levels - 1; l >= 0; --l) {
    if (contains(m->spatial_us, l)) {
      h *= 2; w *= 2;
      if (contains(m->tempo_us, l)) t *= 2;
    }
  }
  if (d.version == 0 && !d.noncausal) t -= d.time_downsample_factor - 1;
  *T = t; *H = h; *W = w;
}

// the fused form of `regularize`: request for the conv_out epilogue (KL: the accumulator is cleared here)
static int make_reg_fusion(vt_model* m, const float* noise, float* z, int32_t* indices, cudaStream_t s, TcRegFusion* rf) {
  const vt_model_desc& d = m->desc;
  *rf = TcRegFusion();
  rf->zc = d.z_channels;
  rf->z = z;
  if (d.regularizer == VT_REG_KL) {
    if (d.kl_sample && !noise) return fail(VT_ERR_INVALID, "KL regularizer with sample=True needs the noise tensor");
    rf->mode = 1; rf->sample = d.kl_sample != 0; rf->noise = noise; rf->kl_acc = m->kl_scratch;
    VT_CUDA(launch_kl_clear(m->kl_scratch, s));
  } else {
    rf->mode = 2; rf->indices = indices;
    for (int i = 0; i < VT_MAX_FSQ && i < d.fsq_num_levels; ++i) rf->fsq_levels[i] = d.fsq_levels[i];
  }
  return VT_OK;
}
static int finish_reg_fusion(vt_model* m, int B, float* kl_loss, cudaStream_t s) {
  if (m->desc.regularizer == VT_REG_KL) VT_CUDA(launch_kl_finish(m->kl_scratch, B, kl_loss, s));
  return VT_OK;
}

static int regularize(vt_model* m, const float* h_pre, const float* noise, int B, int Tz, int Hz, int Wz, float* z,
                      int32_t* indices, float* kl_loss, cudaStream_t s) {
  const vt_model_desc& d = m->desc;
  const long long P = (long long)Tz * Hz * Wz;
  if (d.regularizer == VT_REG_KL) {
    if (d.kl_sample && !noise) return fail(VT_ERR_INVALID, "KL regularizer with sample=True needs the noise tensor");
    VT_CUDA(launch_kl(h_pre, noise, d.z_channels, P, B, d.kl_sample != 0, z, kl_loss, m->kl_scratch, s));
  } else {
    VT_CUDA(launch_fsq(h_pre, d.z_channels, d.fsq_levels, P, B, z, indices, s));
  }
  return VT_OK;
}

}  // namespace vt

// ====================================================================================================
// C ABI
// ====================================================================================================
using namespace vt;

extern "C" {

const char* vt_last_error(void) { return g_err.c_str(); }
int32_t vt_abi_version(void) { return 2; }
int64_t vt_launch_count(int32_t reset) {
  const long long v = g_launches;
  if (reset) g_launches = 0;
  return v;
}

void vt_profile_start(void) { prof_set_detail(false); prof_start(); }
void vt_profile_start_detailed(void) { prof_set_detail(true); prof_start(); }
int32_t vt_profile_stop(char* json, int32_t cap) { return prof_stop(json, cap); }

int32_t vt_model_create(const vt_model_desc* desc, int32_t device, vt_model** out) {
  if (!desc || !out) return fail(VT_ERR_INVALID, "null argument");
  const vt_model_desc& d = *desc;
  if (d.num_levels < 2 || d.num_levels > VT_MAX_LEVELS) return fail(VT_ERR_INVALID, "num_levels out of range");
  if (d.ch <= 0 || d.ch % 4 != 0) return fail(VT_ERR_INVALID, "ch must be a positive multiple of 4");
  if (d.norm_type == VT_NORM_GROUPNORM && d.ch % 32 != 0) return fail(VT_ERR_INVALID, "groupnorm needs ch %% 32 == 0");
  if (d.noncausal && d.version != 0) return fail(VT_ERR_INVALID, "the non-causal family exists in v1.0 only");
  if (d.noncausal && d.norm_type == VT_NORM_GROUPNORM) return fail(VT_ERR_INVALID, "non-causal models with GroupNorm are not on the path (every shipped config uses layernorm)");
  if (d.regularizer == VT_REG_FSQ) {
    if (d.fsq_num_levels != d.z_channels) return fail(VT_ERR_INVALID, "FSQ with projections (dim != len(levels)) is not on the path");
    if (d.double_z) return fail(VT_ERR_INVALID, "FSQ needs double_z = false");
  } else if (!d.double_z) {
    return fail(VT_ERR_INVALID, "KL needs double_z = true");
  }
  vt_model* m = new vt_model();
  m->desc = d;
  m->device = device;
  build_manifest(m);
  *out = m;
  return VT_OK;
}

void vt_model_destroy(vt_model* m) {
  if (!m) return;
  if (m->pool) cudaFree(m->pool);
  if (m->packed_kn) cudaFree(m->packed_kn);
  if (m->packed_nk) cudaFree(m->packed_nk);
  if (m->packed_nk3) cudaFree(m->packed_nk3);
  if (m->packed_stem) cudaFree(m->packed_stem);
  if (m->packed_planes) cudaFree(m->packed_planes);
  if (m->kl_scratch) cudaFree(m->kl_scratch);
  for (auto& kv : m->cache_pool) cudaFree(kv.second);
  if (m->copy_stream) cudaStreamDestroy(m->copy_stream);
  for (int i = 0; i < 2; ++i) {
    if (m->ev_ready[i]) cudaEventDestroy(m->ev_ready[i]);
    if (m->ev_free[i]) cudaEventDestroy(m->ev_free[i]);
    if (m->ev_done[i]) cudaEventDestroy(m->ev_done[i]);
    if (m->ev_drained[i]) cudaEventDestroy(m->ev_drained[i]);
  }
  if (m->ev_join) cudaEventDestroy(m->ev_join);
  delete m;
}

int32_t vt_model_num_params(const vt_model* m) { return m ? (int32_t)m->params.size() : 0; }

int32_t vt_model_param_info(const vt_model* m, int32_t i, char* name, int32_t cap, int64_t* shape5, int32_t* ndim) {
  if (!m || i < 0 || i >= (int)m->params.size()) return fail(VT_ERR_INVALID, "bad parameter index");
  const Param& p = m->params[i];
  if (name && cap > 0) {
    strncpy(name, p.name.c_str(), cap - 1);
    name[cap - 1] = 0;
  }
  if (ndim) *ndim = (int)p.shape.size();
  if (shape5)
    for (size_t k = 0; k < 5; ++k) shape5[k] = k < p.shape.size() ? p.shape[k] : 1;
  return VT_OK;
}

static int ensure_device(vt_model* m) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    return fail(VT_ERR_NO_DEVICE, "no CUDA device visible: vidtok_b200 has no CPU fallback");
  }
  VT_CUDA(cudaSetDevice(m->device));
  if (!m->pool) {
    VT_CUDA(cudaMalloc(&m->pool, (size_t)m->pool_elems * sizeof(float)));
    VT_CUDA(cudaMalloc(&m->kl_scratch, sizeof(double)));
  }
  return VT_OK;
}

int32_t vt_model_load_param(vt_model* m, const char* name, const float* data, int64_t numel, int32_t is_device,
                            void* stream) {
  if (!m || !name || !data) return fail(VT_ERR_INVALID, "null argument");
  auto it = m->index.find(name);
  if (it == m->index.end()) return fail(VT_ERR_INVALID, "unknown parameter %s", name);
  Param& p = m->params[it->second];
  if (p.numel != numel) return fail(VT_ERR_INVALID, "parameter %s: expected %lld elements, got %lld", name, (long long)p.numel, (long long)numel);
  int rc = ensure_device(m);
  if (rc) return rc;
  VT_CUDA(cudaMemcpyAsync(m->pool + p.offset, data, (size_t)numel * sizeof(float),
                          is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, (cudaStream_t)stream));
  p.loaded = true;
  m->finalized = false;
  return VT_OK;
}

int32_t vt_model_finalize(vt_model* m, void* stream) {
  if (!m) return fail(VT_ERR_INVALID, "null model");
  int rc = ensure_device(m);
  if (rc) return rc;
  for (auto& p : m->params)
    if (!p.loaded) return fail(VT_ERR_NOT_READY, "parameter %s was never loaded", p.name.c_str());
  cudaStream_t s = (cudaStream_t)stream;
  // sizes
  size_t kn = 0, nk = 0;
  for (ConvW* c : m->convs) {
    kn += align_up((size_t)c->taps() * c->Ci * c->Co, 64);
    if (c->Kpad) nk += align_up((size_t)c->Co_pad * c->Kpad, 512);
  }
  for (auto& lv : m->dec.levels) {
    if (lv.has_up_phase) nk += 4 * align_up((size_t)lv.up_ph[0].Co_pad * lv.up_ph[0].Kpad, 512);
    if (lv.has_tup_phase) nk += 2 * align_up((size_t)lv.tup_ph[0].Co_pad * lv.tup_ph[0].Kpad, 512);
  }
  if (!m->packed_kn) VT_CUDA(cudaMalloc(&m->packed_kn, kn * sizeof(float)));
  if (!m->packed_nk && nk) VT_CUDA(cudaMalloc(&m->packed_nk, nk * sizeof(bf16)));
  if (!m->packed_nk3 && nk) VT_CUDA(cudaMalloc(&m->packed_nk3, 2 * nk * sizeof(bf16)));   // hi|lo copies (EXACT_TC)
  // power-of-two scales of the split (fp16 hi|lo) weight copies: one max|w| per conv, read back once
  {
    float* d_max = nullptr;
    VT_CUDA(cudaMalloc(&d_max, m->convs.size() * sizeof(float)));
    for (size_t i = 0; i < m->convs.size(); ++i) {
      const ConvW* c = m->convs[i];
      VT_CUDA(launch_absmax(m->pool + m->params[c->pw].offset, (long long)c->Co * c->Ci * c->taps(), d_max + i, s));
    }
    std::vector<float> h_max(m->convs.size());
    cudaError_t e = cudaMemcpyAsync(h_max.data(), d_max, h_max.size() * sizeof(float), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    cudaFree(d_max);
    if (e != cudaSuccess) return fail(VT_ERR_CUDA, "weight scale readback: %s", cudaGetErrorString(e));
    for (size_t i = 0; i < m->convs.size(); ++i) m->convs[i]->wscale3 = split_weight_scale(h_max[i], kModelWeightHeadroom);
  }
  size_t okn = 0, onk = 0;
  for (ConvW* c : m->convs) {
    const int K = c->taps() * c->Ci;
    const float* w = m->pool + m->params[c->pw].offset;
    c->bias = m->pool + m->params[c->pb].offset;
    c->w_kn = m->packed_kn + okn;
    okn += align_up((size_t)K * c->Co, 64);
    VT_CUDA(launch_pack_w_kn(w, c->w_kn, c->Co, c->Ci, c->taps(), s));
    if (c->Kpad) {
      c->w_nk = m->packed_nk + onk;
      c->w_nk3 = m->packed_nk3 + 2 * onk;
      onk += align_up((size_t)c->Co_pad * c->Kpad, 512);
      VT_CUDA(launch_pack_w_nk_bf16(w, c->w_nk, c->Co, c->Co_pad, c->Ci, c->taps(), c->Kpad, s));
      VT_CUDA(launch_pack_w_nk_bf16(w, c->w_nk3, c->Co, c->Co_pad, c->Ci, c->taps(), c->Kpad, s, c->wscale3));
    }
  }
  for (auto& lv : m->dec.levels) {
    const int id3[3] = {0, 1, 2}, id1[3] = {0, 0, 0};
    const int lo[3] = {0, 1, 1}, hi[3] = {0, 0, 1};   // parity 0: taps {0 | 1,2}; parity 1: taps {0,1 | 2}
    if (lv.has_up_phase) {
      const ConvW& c = lv.resample;
      const float* w = m->pool + m->params[c.pw].offset;
      for (int py = 0; py < 2; ++py)
        for (int px = 0; px < 2; ++px) {
          ConvW& ph = lv.up_ph[py * 2 + px];
          ph.bias = c.bias; ph.w_nk = m->packed_nk + onk; ph.w_nk3 = m->packed_nk3 + 2 * onk; ph.wscale3 = c.wscale3;
          onk += align_up((size_t)ph.Co_pad * ph.Kpad, 512);
          VT_CUDA(launch_pack_w_collapsed(w, ph.w_nk, c.Co, c.Co, c.Ci, 1, 3, 3, id1, py == 0 ? lo : hi, px == 0 ? lo : hi, 1, 2, 2, s));
          VT_CUDA(launch_pack_w_collapsed(w, ph.w_nk3, c.Co, c.Co, c.Ci, 1, 3, 3, id1, py == 0 ? lo : hi, px == 0 ? lo : hi, 1, 2, 2, s, c.wscale3));
        }
    }
    if (lv.has_tup_phase) {
      const ConvW& c = lv.tconv;
      const float* w = m->pool + m->params[c.pw].offset;
      for (int pt = 0; pt < 2; ++pt) {
        ConvW& ph = lv.tup_ph[pt];
        ph.bias = c.bias; ph.w_nk = m->packed_nk + onk; ph.w_nk3 = m->packed_nk3 + 2 * onk; ph.wscale3 = c.wscale3;
        onk += align_up((size_t)ph.Co_pad * ph.Kpad, 512);
        // even frames t'=2i read x'[2i-2..2i] = x[i-1],x[i-1],x[i]; odd frames read x[i-1],x[i],x[i]
        // non-causal (pad 1 on both sides): even frames read x'[2i-1..2i+1] = x[i-1],x[i],x[i]; odd frames x[i],x[i],x[i+1]
        const int* tmap = m->desc.noncausal ? (pt == 0 ? lo : hi) : (pt == 0 ? hi : lo);
        VT_CUDA(launch_pack_w_collapsed(w, ph.w_nk, c.Co, c.Co, c.Ci, 3, 3, 3, tmap, id3, id3, 2, 3, 3, s));
        VT_CUDA(launch_pack_w_collapsed(w, ph.w_nk3, c.Co, c.Co, c.Ci, 3, 3, 3, tmap, id3, id3, 2, 3, 3, s, c.wscale3));
      }
    }
  }
  {
    ConvW& c = m->enc.conv_in;
    if (c.stem) {
      if (!m->packed_stem) VT_CUDA(cudaMalloc(&m->packed_stem, (size_t)c.Co * 128 * 3 * sizeof(bf16)));
      c.w_stem = m->packed_stem;
      c.w_stem3 = m->packed_stem + (size_t)c.Co * 128;
      VT_CUDA(launch_pack_w_nk_bf16(m->pool + m->params[c.pw].offset, c.w_stem, c.Co, c.Co, c.Ci, 27, 128, s));
      VT_CUDA(launch_pack_w_nk_bf16(m->pool + m->params[c.pw].offset, c.w_stem3, c.Co, c.Co, c.Ci, 27, 128, s, c.wscale3));
    }
  }
  if (m->head_planes.Kpad) {
    const ConvW& c = m->dec.conv_out;
    if (!m->packed_planes) VT_CUDA(cudaMalloc(&m->packed_planes, (size_t)128 * c.Ci * sizeof(bf16)));
    VT_CUDA(launch_pack_w_tap_planes(m->pool + m->params[c.pw].offset, m->packed_planes, c.Co, c.Ci, 128, s));
    m->head_planes.w_nk = m->packed_planes;
  }
  for (NormW* n : m->norms) {
    n->gamma = m->pool + m->params[n->pg].offset;
    n->beta = m->pool + m->params[n->pb].offset;
  }
  VT_CUDA(cudaStreamSynchronize(s));
  auto set_alpha = [&](LevelW& lv) -> int {
    if (!lv.has_tres) return VT_OK;
    float mix = 0.f;
    VT_CUDA(cudaMemcpy(&mix, m->pool + m->params[lv.p_mix].offset, sizeof(float), cudaMemcpyDeviceToHost));
    lv.alpha = 1.0f / (1.0f + expf(-mix));  // torch.sigmoid(self.mix_factor), model_3dcausal.py:248,268
    return VT_OK;
  };
  for (auto& lv : m->enc.levels) { rc = set_alpha(lv); if (rc) return rc; }
  for (auto& lv : m->dec.levels) { rc = set_alpha(lv); if (rc) return rc; }
  m->finalized = true;
  return VT_OK;
}

int32_t vt_latent_shape(const vt_model* m, int32_t T, int32_t H, int32_t W, int32_t* Tz, int32_t* Hz, int32_t* Wz) {
  if (!m || !Tz || !Hz || !Wz) return fail(VT_ERR_INVALID, "null argument");
  return latent_shape(m, T, H, W, Tz, Hz, Wz);
}
int32_t vt_decoded_frames(const vt_model* m, int32_t Tz) {
  int t, h, w;
  decoded_shape(m, Tz, 1, 1, &t, &h, &w);
  return t;
}

static int spatial_factor(const vt_model* m) {
  int f = 1;
  for (int l = 0; l < m->desc.num_levels; ++l)
    if (contains(m->spatial_ds, l)) f *= 2;
  return f;
}
static int check_hw(const vt_model* m, int H, int W) {
  const int f = spatial_factor(m);
  if (H % f != 0 || W % f != 0) return fail(VT_ERR_INVALID, "H and W must be multiples of %d", f);
  return VT_OK;
}
// what every encode entry point checks of its model and input
static int check_encode_input(const vt_model* m, int C) {
  if (!m->finalized) return fail(VT_ERR_NOT_READY, "vt_model_finalize has not been called");
  if (C != m->desc.in_channels) return fail(VT_ERR_INVALID, "input has %d channels, the model expects in_channels = %d", C, m->desc.in_channels);
  return VT_OK;
}
// ... and every decode entry point (token indices have no channel axis)
static int check_decode_input(const vt_model* m, int Cz, bool from_indices = false) {
  if (!m->finalized) return fail(VT_ERR_NOT_READY, "vt_model_finalize has not been called");
  if (!from_indices && Cz != m->desc.z_channels) return fail(VT_ERR_INVALID, "latent has %d channels, the model expects z_channels = %d", Cz, m->desc.z_channels);
  return VT_OK;
}
// v1.0 streams: the whole clip's time padding is replicated tdf-1 frames, then stride-2 resampling, so the first chunk
// must have 1 (mod tdf) frames and later chunks whole groups of tdf frames
static int check_stream_chunk(const vt_model* m, bool first, int Tc) {
  if (m->desc.version != 0) return VT_OK;
  const int tdf = m->desc.time_downsample_factor;
  if (first ? (Tc % tdf != 1 % tdf) : (Tc % tdf != 0))
    return fail(VT_ERR_INVALID, "a v1.0 stream takes 1 (mod %d) frames in its first chunk and multiples of %d after it, got %d", tdf, tdf, Tc);
  if (first && Tc + (tdf - 1) < 2) return fail(VT_ERR_INVALID, "the first chunk of a v1.0 stream needs two padded frames");
  return VT_OK;
}

static int check_precision(int precision) {
  if (precision < 0 || precision > VT_PREC_MIXED) return fail(VT_ERR_INVALID, "unknown precision mode %d", precision);
  return VT_OK;
}

int64_t vt_workspace_bytes(const vt_model* m, int32_t precision, int32_t B, int32_t T, int32_t H, int32_t W) {
  if (!m || B <= 0 || T <= 0) { fail(VT_ERR_INVALID, "bad shape"); return -1; }
  if (check_precision(precision)) return -1;
  if (check_hw(m, H, W)) return -1;
  vt_model* mm = const_cast<vt_model*>(m);
  int Tz, Hz, Wz;
  latent_shape(m, T, H, W, &Tz, &Hz, &Wz);
  size_t peak = 0;
  {
    Exec ex(mm, stack_prec(precision, false), 0, nullptr, 0, true);
    vt_chunk_state one; one.m = mm; one.persist = false; one.first = true;
    if (m->desc.version == 1) ex.ck = &one;
    float* hpre = (float*)ex.alloc((size_t)B * (m->desc.double_z ? 2 : 1) * m->desc.z_channels * Tz * Hz * Wz * sizeof(float));
    (void)hpre;
    run_encoder(ex, (const float*)(uintptr_t)0x1000, B, T, H, W, (float*)(uintptr_t)0x1000);
    if (!ex.ok()) return -1;
    peak = std::max(peak, ex.ar.peak);
  }
  {
    Exec ex(mm, stack_prec(precision, true), 0, nullptr, 0, true);
    vt_chunk_state one; one.m = mm; one.persist = false; one.first = true; one.is_decoder = true;
    if (m->desc.version == 1) ex.ck = &one;
    float* zc = (float*)ex.alloc((size_t)B * m->desc.z_channels * Tz * Hz * Wz * sizeof(float));  // codes from indices
    (void)zc;
    run_decoder(ex, (const float*)(uintptr_t)0x1000, B, Tz, Hz, Wz, (float*)(uintptr_t)0x1000);
    if (!ex.ok()) return -1;
    peak = std::max(peak, ex.ar.peak);
  }
  return (int64_t)(peak + 4096);
}

// The body of vt_encode and of each chunk: the encoder, then the regularizer (fused into conv_out's epilogue when that runs on
// the wgmma path).  ex is set up with its stream, workspace and chunk context; h_pre (optional) receives the encoder output
// before the regularizer, fp32 [B,Cz,Tz,Hz,Wz].
static int encode(Exec& ex, const float* x, int B, int T, int H, int W, const float* noise, float* z, int32_t* indices,
                  float* kl_loss, float* h_pre) {
  vt_model* m = ex.m;
  int Tz, Hz, Wz;
  latent_shape(m, T, H, W, &Tz, &Hz, &Wz);
  float* hp = h_pre ? h_pre : (float*)ex.alloc((size_t)B * (m->desc.double_z ? 2 : 1) * m->desc.z_channels * Tz * Hz * Wz * sizeof(float));
  if (!ex.ok()) return ex.rc;
  TcRegFusion rf;
  int rc = make_reg_fusion(m, noise, z, indices, ex.s, &rf);
  if (rc) return rc;
  bool reg_done = false;
  run_encoder(ex, x, B, T, H, W, hp, &rf, h_pre != nullptr, &reg_done);
  if (!ex.ok()) return ex.rc;
  if (reg_done) return finish_reg_fusion(m, B, kl_loss, ex.s);
  return regularize(m, hp, noise, B, Tz, Hz, Wz, z, indices, kl_loss, ex.s);
}

int32_t vt_encode(vt_model* m, int32_t precision, const float* x, int32_t B, int32_t C, int32_t T, int32_t H, int32_t W,
                  const float* noise, float* z, int32_t* indices, float* kl_loss, float* h_pre, void* workspace,
                  int64_t workspace_bytes, void* stream) {
  if (!m || !x || !z) return fail(VT_ERR_INVALID, "null argument");
  int rc = check_encode_input(m, C);
  if (rc) return rc;
  if (B <= 0 || T <= 0) return fail(VT_ERR_INVALID, "bad shape");
  rc = check_precision(precision);
  if (rc) return rc;
  rc = check_hw(m, H, W);
  if (rc) return rc;
  VT_CUDA(cudaSetDevice(m->device));
  Exec ex(m, stack_prec(precision, false), (cudaStream_t)stream, workspace, (size_t)workspace_bytes, false);
  vt_chunk_state one; one.m = m; one.persist = false; one.first = true;
  if (m->desc.version == 1) ex.ck = &one;
  return encode(ex, x, B, T, H, W, noise, z, indices, kl_loss, h_pre);
}

int32_t vt_decode(vt_model* m, int32_t precision, const void* z, int32_t from_indices, int32_t B, int32_t Cz, int32_t Tz,
                  int32_t Hz, int32_t Wz, float* x_out, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!m || !z || !x_out) return fail(VT_ERR_INVALID, "null argument");
  if (int rc = check_decode_input(m, Cz, from_indices != 0)) return rc;
  if (B <= 0 || Tz <= 0 || Hz <= 0 || Wz <= 0) return fail(VT_ERR_INVALID, "bad shape");
  if (check_precision(precision)) return VT_ERR_INVALID;
  VT_CUDA(cudaSetDevice(m->device));
  cudaStream_t s = (cudaStream_t)stream;
  Exec ex(m, stack_prec(precision, true), s, workspace, (size_t)workspace_bytes, false);
  vt_chunk_state one; one.m = m; one.persist = false; one.first = true; one.is_decoder = true;
  if (m->desc.version == 1) ex.ck = &one;
  const float* zf = (const float*)z;
  bool idx_in_producer = false;
  if (from_indices) {
    if (m->desc.regularizer != VT_REG_FSQ) return fail(VT_ERR_INVALID, "decode_from_indices needs an FSQ model");
    if (m->desc.version == 0) {
      idx_in_producer = true;   // conv_in forms the codes from the tokens in its gather (no codes tensor)
    } else {
      float* codes = (float*)ex.alloc((size_t)B * m->desc.z_channels * Tz * Hz * Wz * sizeof(float));
      if (!ex.ok()) return ex.rc;
      VT_CUDA(launch_fsq_indices_to_codes((const int*)z, m->desc.z_channels, m->desc.fsq_levels, (long long)Tz * Hz * Wz, B, codes, s));
      zf = codes;
    }
  }
  run_decoder(ex, zf, B, Tz, Hz, Wz, x_out, idx_in_producer);
  return ex.rc;
}

// ---- chunked v1.1 ------------------------------------------------------------------------------------
int32_t vt_chunk_state_create(vt_model* m, int32_t precision, int32_t B, int32_t H, int32_t W, int32_t is_decoder,
                              int32_t use_overlap, vt_chunk_state** out) {
  if (!m || !out) return fail(VT_ERR_INVALID, "null argument");
  if (m->desc.noncausal)
    return fail(VT_ERR_INVALID, "non-causal models cannot stream: their time padding is symmetric, so a frame depends on later frames");
  if (m->desc.version == 0 && use_overlap) return fail(VT_ERR_INVALID, "overlap look-ahead exists only in the v1.1 model family");
  if (check_precision(precision)) return VT_ERR_INVALID;
  if (B <= 0 || H <= 0 || W <= 0) return fail(VT_ERR_INVALID, "bad shape");
  if (check_hw(m, H * (is_decoder ? spatial_factor(m) : 1), W * (is_decoder ? spatial_factor(m) : 1))) return VT_ERR_INVALID;
  vt_chunk_state* st = new vt_chunk_state();
  st->m = m; st->prec = precision; st->B = B; st->H = H; st->W = W;
  st->is_decoder = is_decoder != 0; st->use_overlap = use_overlap != 0;
  st->first = true; st->persist = true;
  *out = st;
  return VT_OK;
}
void vt_chunk_state_destroy(vt_chunk_state* s) { delete s; }

int64_t vt_chunk_workspace_bytes(const vt_chunk_state* cs, int32_t Tc) {
  if (!cs) { fail(VT_ERR_INVALID, "null state"); return -1; }
  vt_chunk_state tmp;  // measure with throw-away cache bookkeeping
  tmp.m = cs->m; tmp.prec = cs->prec; tmp.B = cs->B; tmp.H = cs->H; tmp.W = cs->W;
  tmp.is_decoder = cs->is_decoder; tmp.use_overlap = cs->use_overlap; tmp.persist = true;
  size_t peak = 0;
  for (int first = 0; first < 2; ++first) {
    tmp.first = first != 0;
    Exec ex(cs->m, stack_prec(cs->prec, cs->is_decoder), 0, nullptr, 0, true);
    ex.ck = &tmp;
    if (cs->is_decoder) {
      run_decoder(ex, (const float*)(uintptr_t)0x1000, cs->B, Tc, cs->H, cs->W, (float*)(uintptr_t)0x1000);
    } else {
      int Tz, Hz, Wz;
      latent_shape(cs->m, Tc, cs->H, cs->W, &Tz, &Hz, &Wz);
      ex.alloc((size_t)cs->B * 2 * cs->m->desc.z_channels * Tz * Hz * Wz * sizeof(float));
      run_encoder(ex, (const float*)(uintptr_t)0x1000, cs->B, Tc, cs->H, cs->W, (float*)(uintptr_t)0x1000);
    }
    if (!ex.ok()) return -1;
    peak = std::max(peak, ex.ar.peak);
  }
  return (int64_t)(peak + 4096);
}

// h_out (optional): the chunk's encoder output before the regularizer, fp32 [B,Cz,Tz,Hz,Wz] (the FSQ aux loss reads it)
static int encode_chunk(vt_chunk_state* cs, int32_t is_first, const float* x_chunk, int32_t C, int32_t Tc, const float* noise,
                        float* z, int32_t* indices, float* kl_loss, float* h_out, void* workspace, int64_t workspace_bytes,
                        void* stream) {
  if (!cs || !x_chunk || !z) return fail(VT_ERR_INVALID, "null argument");
  if (cs->is_decoder) return fail(VT_ERR_INVALID, "decoder state passed to vt_encode_chunk");
  vt_model* m = cs->m;
  int rc = check_encode_input(m, C);
  if (rc) return rc;
  VT_CUDA(cudaSetDevice(m->device));
  if (Tc <= 0) return fail(VT_ERR_INVALID, "bad shape");
  rc = check_stream_chunk(m, is_first != 0, Tc);
  if (rc) return rc;
  cs->first = is_first != 0;
  Exec ex(m, stack_prec(cs->prec, false), (cudaStream_t)stream, workspace, (size_t)workspace_bytes, false);
  ex.ck = cs;
  return encode(ex, x_chunk, cs->B, Tc, cs->H, cs->W, noise, z, indices, kl_loss, h_out);
}
int32_t vt_encode_chunk(vt_chunk_state* cs, int32_t is_first, const float* x_chunk, int32_t C, int32_t Tc, const float* noise,
                        float* z, int32_t* indices, float* kl_loss, void* workspace, int64_t workspace_bytes,
                        void* stream) {
  return encode_chunk(cs, is_first, x_chunk, C, Tc, noise, z, indices, kl_loss, nullptr, workspace, workspace_bytes, stream);
}

int32_t vt_decode_chunk(vt_chunk_state* cs, int32_t is_first, const float* z_chunk, int32_t Cz, int32_t Tzc, float* x_out,
                        void* workspace, int64_t workspace_bytes, void* stream) {
  if (!cs || !z_chunk || !x_out) return fail(VT_ERR_INVALID, "null argument");
  if (!cs->is_decoder) return fail(VT_ERR_INVALID, "encoder state passed to vt_decode_chunk");
  vt_model* m = cs->m;
  if (int rc = check_decode_input(m, Cz)) return rc;
  if (Tzc <= 0) return fail(VT_ERR_INVALID, "bad shape");
  VT_CUDA(cudaSetDevice(m->device));
  cs->first = is_first != 0;
  Exec ex(m, stack_prec(cs->prec, true), (cudaStream_t)stream, workspace, (size_t)workspace_bytes, false);
  ex.ck = cs;
  run_decoder(ex, z_chunk, cs->B, Tzc, cs->H, cs->W, x_out);
  return ex.rc;
}

// ---- whole-video temporal tiling in the library (autoencoder_v1_1.py:218-228,244-264,302-331) ------------------------------
// The chunk schedule, the per-layer caches and the chunk staging all live below the ABI: one call per video, no host
// synchronisation, no per-chunk allocation.  Chunk i+1 is staged (host -> device, or a strided device copy) into the second
// staging buffer on the library's copy stream while chunk i computes on the caller's stream (double buffering); decoded
// chunks leave the same way.
namespace {
struct ChunkSpan { int s, e; };
// build_chunk_start_end (autoencoder_v1_1.py:218-228): [0,1], then steps of `step`
std::vector<ChunkSpan> chunk_schedule(int t, int step) {
  std::vector<ChunkSpan> v;
  v.push_back({0, 1});
  int start = 1, end = 1;
  while (start < t) {
    end = std::min(t, end + step);
    v.push_back({start, end});
    start = end;
  }
  return v;
}
int ensure_copy_stream(vt_model* m) {
  if (m->copy_stream) return VT_OK;
  VT_CUDA(cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
  for (int i = 0; i < 2; ++i) {
    VT_CUDA(cudaEventCreateWithFlags(&m->ev_ready[i], cudaEventDisableTiming));
    VT_CUDA(cudaEventCreateWithFlags(&m->ev_free[i], cudaEventDisableTiming));
    VT_CUDA(cudaEventCreateWithFlags(&m->ev_done[i], cudaEventDisableTiming));
    VT_CUDA(cudaEventCreateWithFlags(&m->ev_drained[i], cudaEventDisableTiming));
  }
  VT_CUDA(cudaEventCreateWithFlags(&m->ev_join, cudaEventDisableTiming));
  return VT_OK;
}
__global__ void mean_kernel(const float* v, int n, float* out) {
  float s = 0.f;
  for (int i = 0; i < n; ++i) s += v[i];
  *out = s / (float)n;
}
// frames [t0, t0+n) of a [rows, T, frame] tensor <-> a dense [rows, n, frame] chunk (one strided 2-D copy)
cudaError_t copy_frames_2d(void* dst, size_t dst_T, size_t dst_t0, const void* src, size_t src_T, size_t src_t0, size_t rows, size_t n,
                           size_t frame_bytes, cudaMemcpyKind kind, cudaStream_t s) {
  if (rows == 0 || n == 0) return cudaSuccess;
  return cudaMemcpy2DAsync((char*)dst + dst_t0 * frame_bytes, dst_T * frame_bytes, (const char*)src + src_t0 * frame_bytes,
                           src_T * frame_bytes, n * frame_bytes, rows, kind, s);
}
size_t up1k(size_t n) { return (n + 1023) / 1024 * 1024; }
}  // namespace

static int64_t video_workspace(const vt_model* m, int precision, int B, int T, int H, int W, int t_chunk, bool decoder, bool overlap) {
  // staging + dense per-chunk outputs + the largest chunk workspace.  T/H/W: input video (encoder) or latent geometry (decoder).
  vt_chunk_state tmp;
  tmp.m = const_cast<vt_model*>(m); tmp.prec = precision; tmp.B = B; tmp.H = H; tmp.W = W;
  tmp.is_decoder = decoder; tmp.use_overlap = overlap; tmp.persist = true;
  const vt_model_desc& d = m->desc;
  size_t fixed = 0, peak = 0;
  std::vector<int> lens;
  for (const ChunkSpan& c : chunk_schedule(T, t_chunk)) {
    int n = c.e - c.s + ((decoder && overlap && c.e + 1 <= T) ? 1 : 0);
    if (std::find(lens.begin(), lens.end(), n) == lens.end()) lens.push_back(n);
  }
  int max_len = *std::max_element(lens.begin(), lens.end());
  if (!decoder) {
    int Tz, Hz, Wz;
    latent_shape(m, max_len, H, W, &Tz, &Hz, &Wz);
    fixed += 2 * up1k((size_t)B * d.in_channels * max_len * H * W * 4);           // input staging x 2
    fixed += 2 * up1k((size_t)B * d.z_channels * Tz * Hz * Wz * 4) + up1k((size_t)B * Tz * Hz * Wz * 4);   // noise, z, indices (dense chunk)
    fixed += up1k(4096);                                                            // per-chunk kl values
  } else {
    int To, Ho, Wo;
    decoded_shape(m, max_len, H, W, &To, &Ho, &Wo);
    fixed += up1k((size_t)B * d.z_channels * max_len * H * W * 4);                 // dense latent chunk
    fixed += 2 * up1k((size_t)B * d.out_ch * To * Ho * Wo * 4);                    // decoded chunk x 2
  }
  for (int n : lens) {
    const int64_t w = vt_chunk_workspace_bytes(&tmp, n);
    if (w < 0) return -1;
    peak = std::max(peak, (size_t)w);
  }
  return (int64_t)(fixed + peak + 8192);
}

int64_t vt_encode_video_workspace_bytes(const vt_model* m, int32_t precision, int32_t B, int32_t T, int32_t H, int32_t W,
                                        int32_t t_chunk_enc) {
  if (!m || B <= 0 || T <= 0 || t_chunk_enc <= 0) { fail(VT_ERR_INVALID, "bad shape"); return -1; }
  if (m->desc.version != 1) { fail(VT_ERR_INVALID, "temporal tiling exists only in the v1.1 model family"); return -1; }
  if (check_precision(precision) || check_hw(m, H, W)) return -1;
  return video_workspace(m, precision, B, T, H, W, t_chunk_enc, false, false);
}
int64_t vt_decode_video_workspace_bytes(const vt_model* m, int32_t precision, int32_t B, int32_t Tz, int32_t Hz, int32_t Wz,
                                        int32_t t_chunk_dec, int32_t use_overlap) {
  if (!m || B <= 0 || Tz <= 0 || t_chunk_dec <= 0) { fail(VT_ERR_INVALID, "bad shape"); return -1; }
  if (m->desc.version != 1) { fail(VT_ERR_INVALID, "temporal tiling exists only in the v1.1 model family"); return -1; }
  if (check_precision(precision)) return -1;
  return video_workspace(m, precision, B, Tz, Hz, Wz, t_chunk_dec, true, use_overlap != 0);
}
// frames vt_decode_video writes: per chunk vt_decoded_frames(len) minus the dropped look-ahead tail (autoencoder_v1_1.py:327-328)
int32_t vt_decode_video_frames(const vt_model* m, int32_t Tz, int32_t t_chunk_dec, int32_t use_overlap) {
  if (!m || Tz <= 0 || t_chunk_dec <= 0) return -1;
  const int tdf = m->desc.time_downsample_factor;
  int total = 0;
  for (const ChunkSpan& c : chunk_schedule(Tz, t_chunk_dec)) {
    const bool look = use_overlap && c.e + 1 <= Tz;
    total += vt_decoded_frames(m, c.e - c.s + (look ? 1 : 0)) - (look ? tdf : 0);
  }
  return total;
}

// FSQ aux-loss partials of every chunk (vt_encode_video_fsq_aux): chunk i writes stats[2i..2i+1] and avg_prob[i*J ..)
namespace {
struct VideoAux {
  float inv_t;
  float* stats;
  float* avg_prob;
};
// latent tokens of the longest chunk (the aux workspace is sized for it)
long long video_max_chunk_tokens(const vt_model* m, int B, int T, int H, int W, int t_chunk) {
  long long best = 0;
  for (const ChunkSpan& c : chunk_schedule(T, t_chunk)) {
    int Tz, Hz, Wz;
    latent_shape(m, c.e - c.s, H, W, &Tz, &Hz, &Wz);
    best = std::max(best, (long long)B * Tz * Hz * Wz);
  }
  return best;
}
// what a chunk's aux partials write and read: stats [2], avg_prob [J], the pre-bound latent h fp32 [B,Cz,Tz,Hz,Wz] and the
// partials' scratch (fsq_aux_workspace of the chunk's tokens)
struct ChunkAux {
  float inv_t;
  float* stats;
  float* avg_prob;
  float* h;
  void* ws;
};
}  // namespace

// One chunk of an encode stream or of vt_encode_video: the encoder and the regularizer, then (aux != NULL) the FSQ aux
// partials of the chunk's tokens from its pre-bound latent.  The aux geometry is checked before anything is launched.
static int encode_chunk_aux(vt_chunk_state* cs, int32_t is_first, const float* x_chunk, int32_t C, int32_t Tc, const float* noise,
                            float* z, int32_t* indices, float* kl_loss, const ChunkAux* aux, void* workspace, int64_t workspace_bytes,
                            void* stream) {
  FsqAuxGeom ag;
  long long P = 0;
  if (aux) {
    if (!cs) return fail(VT_ERR_INVALID, "null argument");
    const vt_model_desc& d = cs->m->desc;
    if (d.regularizer != VT_REG_FSQ) return fail(VT_ERR_INVALID, "the FSQ aux loss needs an FSQ model");
    if (Tc <= 0) return fail(VT_ERR_INVALID, "bad shape");
    int Tz, Hz, Wz;
    latent_shape(cs->m, Tc, cs->H, cs->W, &Tz, &Hz, &Wz);
    P = (long long)Tz * Hz * Wz;
    const char* why = fsq_aux_geometry(d.z_channels, d.fsq_levels, (long long)cs->B * P, &ag);
    if (why) return fail(VT_ERR_INVALID, "%s", why);
  }
  int rc = encode_chunk(cs, is_first, x_chunk, C, Tc, noise, z, indices, kl_loss, aux ? aux->h : nullptr, workspace, workspace_bytes,
                        stream);
  if (rc || !aux) return rc;
  VT_CUDA(launch_fsq_aux_partials(aux->h, ag, cs->m->desc.fsq_levels, P, aux->inv_t, aux->stats, aux->avg_prob, aux->ws,
                                  (cudaStream_t)stream));
  return VT_OK;
}

static int encode_video(vt_model* m, int32_t precision, const float* x, int32_t x_on_host, int32_t B, int32_t C, int32_t T,
                        int32_t H, int32_t W, int32_t t_chunk_enc, const float* noise, float* z, int32_t* indices,
                        float* kl_loss, const VideoAux* aux, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!m || !x || !z || !workspace) return fail(VT_ERR_INVALID, "null argument");
  if (m->desc.version != 1) return fail(VT_ERR_INVALID, "temporal tiling exists only in the v1.1 model family");
  int rc = check_encode_input(m, C);
  if (rc) return rc;
  if (B <= 0 || T <= 0 || t_chunk_enc <= 0) return fail(VT_ERR_INVALID, "bad shape");
  rc = check_precision(precision);
  if (rc) return rc;
  rc = check_hw(m, H, W);
  if (rc) return rc;
  VT_CUDA(cudaSetDevice(m->device));
  rc = ensure_copy_stream(m);
  if (rc) return rc;
  const vt_model_desc& d = m->desc;
  cudaStream_t s = (cudaStream_t)stream, cs = m->copy_stream;
  const std::vector<ChunkSpan> chunks = chunk_schedule(T, t_chunk_enc);
  int max_len = 0, TzTot = 0;
  std::vector<int> tz_of(chunks.size());
  int Hz = 0, Wz = 0;
  for (size_t i = 0; i < chunks.size(); ++i) {
    max_len = std::max(max_len, chunks[i].e - chunks[i].s);
    latent_shape(m, chunks[i].e - chunks[i].s, H, W, &tz_of[i], &Hz, &Wz);
    TzTot += tz_of[i];
  }
  if ((int)chunks.size() > 1024) return fail(VT_ERR_INVALID, "too many chunks");
  int TzMax, hz_, wz_;
  latent_shape(m, max_len, H, W, &TzMax, &hz_, &wz_);
  // carve the workspace
  char* w = (char*)workspace;
  const size_t stage_b = up1k((size_t)B * C * max_len * H * W * 4), lat_b = up1k((size_t)B * d.z_channels * TzMax * Hz * Wz * 4);
  float* stage[2] = {(float*)w, (float*)(w + stage_b)};
  w += 2 * stage_b;
  float* noise_c = (float*)w; w += lat_b;
  float* z_c = (float*)w; w += lat_b;
  int32_t* idx_c = (int32_t*)w; w += up1k((size_t)B * TzMax * Hz * Wz * 4);
  float* kl_c = (float*)w; w += up1k(4096);
  float* h_c = nullptr;
  void* aux_ws = nullptr;
  FsqAuxGeom ag;
  if (aux) {
    if (d.regularizer != VT_REG_FSQ) return fail(VT_ERR_INVALID, "the FSQ aux loss needs an FSQ model");
    const char* why = fsq_aux_geometry(d.z_channels, d.fsq_levels, video_max_chunk_tokens(m, B, T, H, W, t_chunk_enc), &ag);
    if (why) return fail(VT_ERR_INVALID, "%s", why);
    h_c = (float*)w; w += lat_b;
    aux_ws = w; w += up1k(fsq_aux_workspace(ag));
  }
  const int64_t ws_left = workspace_bytes - (w - (char*)workspace);
  if (ws_left <= 0) return fail(VT_ERR_WORKSPACE, "workspace too small for the chunk staging buffers");
  const size_t fr_in = (size_t)H * W * 4, fr_z = (size_t)Hz * Wz * 4;
  const cudaMemcpyKind in_kind = x_on_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
  // the copy stream must not start staging before the caller's stream has produced x / released the workspace
  VT_CUDA(cudaEventRecord(m->ev_join, s));
  VT_CUDA(cudaStreamWaitEvent(cs, m->ev_join, 0));
  vt_chunk_state* st = nullptr;
  rc = vt_chunk_state_create(m, precision, B, H, W, 0, 0, &st);
  if (rc) return rc;
  auto stage_chunk = [&](size_t i) -> cudaError_t {
    const int n = chunks[i].e - chunks[i].s;
    cudaError_t e = copy_frames_2d(stage[i & 1], n, 0, x, T, chunks[i].s, (size_t)B * C, n, fr_in, in_kind, cs);
    if (e == cudaSuccess) e = cudaEventRecord(m->ev_ready[i & 1], cs);
    return e;
  };
  cudaError_t ce = stage_chunk(0);
  int tz0 = 0;
  for (size_t i = 0; i < chunks.size() && ce == cudaSuccess && rc == VT_OK; ++i) {
    const int cur = (int)(i & 1), n = chunks[i].e - chunks[i].s, tzc = tz_of[i];
    if (i + 1 < chunks.size()) {
      if (i >= 1) ce = cudaStreamWaitEvent(cs, m->ev_free[cur ^ 1], 0);   // chunk i-1 (which read that buffer) has finished
      if (ce == cudaSuccess) ce = stage_chunk(i + 1);
    }
    if (ce == cudaSuccess) ce = cudaStreamWaitEvent(s, m->ev_ready[cur], 0);
    if (ce == cudaSuccess && noise)
      ce = copy_frames_2d(noise_c, tzc, 0, noise, TzTot, tz0, (size_t)B * d.z_channels, tzc, fr_z, cudaMemcpyDeviceToDevice, s);
    if (ce != cudaSuccess) break;
    const ChunkAux ca{aux ? aux->inv_t : 0.f, aux ? aux->stats + 2 * i : nullptr, aux ? aux->avg_prob + (size_t)i * ag.J : nullptr,
                      h_c, aux_ws};
    rc = encode_chunk_aux(st, i == 0, stage[cur], C, n, noise ? noise_c : nullptr, z_c, indices ? idx_c : nullptr,
                          d.regularizer == VT_REG_KL ? kl_c + i : nullptr, aux ? &ca : nullptr, w, ws_left, stream);
    if (rc) break;
    ce = cudaEventRecord(m->ev_free[cur], s);
    if (ce == cudaSuccess) ce = copy_frames_2d(z, TzTot, tz0, z_c, tzc, 0, (size_t)B * d.z_channels, tzc, fr_z, cudaMemcpyDeviceToDevice, s);
    if (ce == cudaSuccess && indices)
      ce = copy_frames_2d(indices, TzTot, tz0, idx_c, tzc, 0, (size_t)B, tzc, fr_z, cudaMemcpyDeviceToDevice, s);
    tz0 += tzc;
  }
  if (ce == cudaSuccess && rc == VT_OK && d.regularizer == VT_REG_KL && kl_loss) {
    mean_kernel<<<1, 1, 0, s>>>(kl_c, (int)chunks.size(), kl_loss);   // torch.mean(torch.stack(kls)), autoencoder_v1_1.py:261-264
    count_launch();
    ce = cudaGetLastError();
  }
  // the caller's stream owns the workspace again only after the copy stream has drained
  cudaEventRecord(m->ev_join, cs);
  cudaStreamWaitEvent(s, m->ev_join, 0);
  vt_chunk_state_destroy(st);
  if (rc) return rc;
  if (ce != cudaSuccess) return fail(VT_ERR_CUDA, "vt_encode_video: %s", cudaGetErrorString(ce));
  return VT_OK;
}

int32_t vt_encode_video(vt_model* m, int32_t precision, const float* x, int32_t x_on_host, int32_t B, int32_t C, int32_t T,
                        int32_t H, int32_t W, int32_t t_chunk_enc, const float* noise, float* z, int32_t* indices,
                        float* kl_loss, void* workspace, int64_t workspace_bytes, void* stream) {
  return encode_video(m, precision, x, x_on_host, B, C, T, H, W, t_chunk_enc, noise, z, indices, kl_loss, nullptr, workspace,
                      workspace_bytes, stream);
}

int64_t vt_encode_video_fsq_aux_workspace_bytes(const vt_model* m, int32_t precision, int32_t B, int32_t T, int32_t H, int32_t W,
                                                int32_t t_chunk_enc) {
  const int64_t base = vt_encode_video_workspace_bytes(m, precision, B, T, H, W, t_chunk_enc);
  if (base < 0) return -1;
  const vt_model_desc& d = m->desc;
  if (d.regularizer != VT_REG_FSQ) { fail(VT_ERR_INVALID, "the FSQ aux loss needs an FSQ model"); return -1; }
  int max_len = 0;
  for (const ChunkSpan& c : chunk_schedule(T, t_chunk_enc)) max_len = std::max(max_len, c.e - c.s);
  int TzMax, Hz, Wz;
  latent_shape(m, max_len, H, W, &TzMax, &Hz, &Wz);
  FsqAuxGeom ag;
  const char* why = fsq_aux_geometry(d.z_channels, d.fsq_levels, video_max_chunk_tokens(m, B, T, H, W, t_chunk_enc), &ag);
  if (why) { fail(VT_ERR_INVALID, "%s", why); return -1; }
  return base + (int64_t)up1k((size_t)B * d.z_channels * TzMax * Hz * Wz * 4) + (int64_t)up1k(fsq_aux_workspace(ag));
}

int32_t vt_encode_video_fsq_aux(vt_model* m, int32_t precision, const float* x, int32_t x_on_host, int32_t B, int32_t C, int32_t T,
                                int32_t H, int32_t W, int32_t t_chunk_enc, float* z, int32_t* indices, float inv_temperature,
                                float* aux_stats, float* aux_avg_prob, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!aux_stats || !aux_avg_prob) return fail(VT_ERR_INVALID, "null argument");
  const VideoAux aux{inv_temperature, aux_stats, aux_avg_prob};
  return encode_video(m, precision, x, x_on_host, B, C, T, H, W, t_chunk_enc, nullptr, z, indices, nullptr, &aux, workspace,
                      workspace_bytes, stream);
}

// vt_encode_chunk_fsq_aux's workspace: [h | aux scratch | vt_chunk_workspace_bytes]
static int chunk_aux_layout(const vt_chunk_state* cs, int32_t Tc, size_t* h_bytes, size_t* aux_bytes) {
  if (!cs) return fail(VT_ERR_INVALID, "null state");
  if (cs->is_decoder) return fail(VT_ERR_INVALID, "decoder state passed to vt_encode_chunk_fsq_aux");
  const vt_model_desc& d = cs->m->desc;
  if (d.regularizer != VT_REG_FSQ) return fail(VT_ERR_INVALID, "the FSQ aux loss needs an FSQ model");
  if (Tc <= 0) return fail(VT_ERR_INVALID, "bad shape");
  int Tz, Hz, Wz;
  latent_shape(cs->m, Tc, cs->H, cs->W, &Tz, &Hz, &Wz);
  FsqAuxGeom ag;
  const char* why = fsq_aux_geometry(d.z_channels, d.fsq_levels, (long long)cs->B * Tz * Hz * Wz, &ag);
  if (why) return fail(VT_ERR_INVALID, "%s", why);
  *h_bytes = up1k((size_t)cs->B * d.z_channels * Tz * Hz * Wz * 4);
  *aux_bytes = up1k(fsq_aux_workspace(ag));
  return VT_OK;
}

int64_t vt_chunk_fsq_aux_workspace_bytes(const vt_chunk_state* cs, int32_t Tc) {
  size_t hb, ab;
  if (chunk_aux_layout(cs, Tc, &hb, &ab)) return -1;
  const int64_t base = vt_chunk_workspace_bytes(cs, Tc);
  if (base < 0) return -1;
  return (int64_t)(hb + ab) + base;
}

int32_t vt_encode_chunk_fsq_aux(vt_chunk_state* cs, int32_t is_first, const float* x_chunk, int32_t C, int32_t Tc, float* z,
                                int32_t* indices, float inv_temperature, float* stats, float* avg_prob, void* workspace,
                                int64_t workspace_bytes, void* stream) {
  size_t hb, ab;
  if (int rc = chunk_aux_layout(cs, Tc, &hb, &ab)) return rc;
  if (!stats || !avg_prob || !workspace) return fail(VT_ERR_INVALID, "null argument");
  if (workspace_bytes <= (int64_t)(hb + ab)) return fail(VT_ERR_WORKSPACE, "workspace too small for the FSQ aux loss");
  char* w = (char*)workspace;
  const ChunkAux aux{inv_temperature, stats, avg_prob, (float*)w, w + hb};
  return encode_chunk_aux(cs, is_first, x_chunk, C, Tc, nullptr, z, indices, nullptr, &aux, w + hb + ab,
                          workspace_bytes - (int64_t)(hb + ab), stream);
}

int32_t vt_decode_video(vt_model* m, int32_t precision, const float* z, int32_t B, int32_t Cz, int32_t Tz, int32_t Hz, int32_t Wz,
                        int32_t t_chunk_dec, int32_t use_overlap, float* x_out, int32_t out_on_host, void* workspace,
                        int64_t workspace_bytes, void* stream) {
  if (!m || !z || !x_out || !workspace) return fail(VT_ERR_INVALID, "null argument");
  if (m->desc.version != 1) return fail(VT_ERR_INVALID, "temporal tiling exists only in the v1.1 model family");
  int rc = check_decode_input(m, Cz);
  if (rc) return rc;
  if (B <= 0 || Tz <= 0 || t_chunk_dec <= 0) return fail(VT_ERR_INVALID, "bad shape");
  rc = check_precision(precision);
  if (rc) return rc;
  const vt_model_desc& d = m->desc;
  const int tdf = d.time_downsample_factor;
  if (use_overlap && tdf != 2 && tdf != 4 && tdf != 8) return fail(VT_ERR_INVALID, "use_overlap supports 2x, 4x or 8x temporal downsampling only");
  VT_CUDA(cudaSetDevice(m->device));
  rc = ensure_copy_stream(m);
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream, cs = m->copy_stream;
  const std::vector<ChunkSpan> chunks = chunk_schedule(Tz, t_chunk_dec);
  int max_len = 0;
  for (const ChunkSpan& c : chunks) max_len = std::max(max_len, c.e - c.s + ((use_overlap && c.e + 1 <= Tz) ? 1 : 0));
  int ToMax, Ho, Wo;
  decoded_shape(m, max_len, Hz, Wz, &ToMax, &Ho, &Wo);
  const int T_out = vt_decode_video_frames(m, Tz, t_chunk_dec, use_overlap);
  char* w = (char*)workspace;
  float* z_c = (float*)w; w += up1k((size_t)B * Cz * max_len * Hz * Wz * 4);
  const size_t out_b = up1k((size_t)B * d.out_ch * ToMax * Ho * Wo * 4);
  float* out_c[2] = {(float*)w, (float*)(w + out_b)};
  w += 2 * out_b;
  const int64_t ws_left = workspace_bytes - (w - (char*)workspace);
  if (ws_left <= 0) return fail(VT_ERR_WORKSPACE, "workspace too small for the chunk staging buffers");
  const size_t fr_z = (size_t)Hz * Wz * 4, fr_o = (size_t)Ho * Wo * 4;
  const cudaMemcpyKind out_kind = out_on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  vt_chunk_state* st = nullptr;
  rc = vt_chunk_state_create(m, precision, B, Hz, Wz, 1, use_overlap, &st);
  if (rc) return rc;
  cudaError_t ce = cudaSuccess;
  int t0 = 0;
  for (size_t i = 0; i < chunks.size() && ce == cudaSuccess && rc == VT_OK; ++i) {
    const int cur = (int)(i & 1);
    const bool look = use_overlap && chunks[i].e + 1 <= Tz;
    const int n = chunks[i].e - chunks[i].s + (look ? 1 : 0);
    const int To = vt_decoded_frames(m, n), keep = To - (look ? tdf : 0);
    ce = copy_frames_2d(z_c, n, 0, z, Tz, chunks[i].s, (size_t)B * Cz, n, fr_z, cudaMemcpyDeviceToDevice, s);
    if (ce == cudaSuccess && i >= 2) ce = cudaStreamWaitEvent(s, m->ev_drained[cur], 0);   // chunk i-2 has left this buffer
    if (ce != cudaSuccess) break;
    rc = vt_decode_chunk(st, i == 0, z_c, Cz, n, out_c[cur], w, ws_left, stream);
    if (rc) break;
    // the decoded chunk leaves on the copy stream (device -> host, or into the caller's device tensor) while the next one computes
    ce = cudaEventRecord(m->ev_done[cur], s);
    if (ce == cudaSuccess) ce = cudaStreamWaitEvent(cs, m->ev_done[cur], 0);
    if (ce == cudaSuccess) ce = copy_frames_2d(x_out, T_out, t0, out_c[cur], To, 0, (size_t)B * d.out_ch, keep, fr_o, out_kind, cs);
    if (ce == cudaSuccess) ce = cudaEventRecord(m->ev_drained[cur], cs);
    t0 += keep;
  }
  cudaEventRecord(m->ev_join, cs);
  cudaStreamWaitEvent(s, m->ev_join, 0);
  vt_chunk_state_destroy(st);
  if (rc) return rc;
  if (ce != cudaSuccess) return fail(VT_ERR_CUDA, "vt_decode_video: %s", cudaGetErrorString(ce));
  return VT_OK;
}

// ---- single operators (parity tests) -----------------------------------------------------------------
static inline DType act_type(int precision) {
  return precision == VT_PREC_FMA32 ? DT_F32 : (precision == VT_PREC_EXACT_TC ? DT_SPLIT : DT_BF16);
}

// power-of-two scale of the split copy of an operator's weight tensor (the model path does this once in vt_model_finalize)
static int op_weight_scale(const float* w, long long n, float headroom, cudaStream_t s, float* scale) {
  float* d_max = nullptr;
  VT_CUDA(cudaMalloc(&d_max, sizeof(float)));
  float h = 0.f;
  cudaError_t e = launch_absmax(w, n, d_max, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&h, d_max, sizeof(float), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  cudaFree(d_max);
  if (e != cudaSuccess) return fail(VT_ERR_CUDA, "weight scale: %s", cudaGetErrorString(e));
  *scale = split_weight_scale(h, headroom);
  return VT_OK;
}

// Shared body of vt_op_conv / vt_op_conv_ex: one convolution launch of the kernel the model path uses for that
// precision, with temporary weight repacks.
static int op_conv_impl(int precision, int force_simt, const vt_conv_desc* d, const vt_conv_ex* e, const void* x,
                        const void* cache, const float* w, const float* bias, const void* res, const float* gamma,
                        const float* beta, void* out, void* out2, cudaStream_t s, const TcRegFusion* reg = nullptr,
                        bool relu = false) {
  if (!d || !x || !w || (!out && !reg)) return fail(VT_ERR_INVALID, "null argument");
  if (precision != VT_PREC_FMA32 && precision != VT_PREC_BF16 && precision != VT_PREC_EXACT_TC)
    return fail(VT_ERR_INVALID, "operator precision must be FMA32, BF16 or EXACT_TC");
  const DType ta = act_type(precision);
  const long long cw = ta == DT_SPLIT ? 2 : 1;
  ConvP p = conv_p(d->B, d->Ti, d->Hi, d->Wi, d->Ci);
  p.split = ta == DT_SPLIT ? 1 : 0;
  set_in(p, cl_strides(d->Ti, d->Hi, d->Wi, d->Ci, cw));
  p.kt = d->kt; p.kh = d->kh; p.kw = d->kw; p.st = d->st; p.sh = d->sh; p.sw = d->sw;
  p.ut = d->ut; p.uh = d->uh; p.uw = d->uw;
  p.pt = d->pt; p.ph = d->ph0; p.pw = d->pw0;
  p.to_off = e ? e->to_off : 0;
  p.Co = d->Co;
  if (!conv_out_size(p, 0, d->ph1, d->pw1)) return fail(VT_ERR_INVALID, "conv: empty output");
  const bool out_f32 = e && e->out_f32_ncdhw;
  // out_f32: external fp32 [B,Co,To,Ho,Wo] (the heads)
  set_out(p, out_f32 ? ncdhw_strides(p.Co, p.To, p.Ho, p.Wo) : cl_strides(p.To, p.Ho, p.Wo, p.Co, cw));
  if (e && e->t_mode) {
    if (e->t_mode == 2 && (!cache || e->cacheT <= 0)) return fail(VT_ERR_INVALID, "t_mode 2 needs a cache of cacheT frames");
    p.t_mode = e->t_mode; p.cache = cache; p.cacheT = e->cacheT;
  }
  p.bias = bias;
  p.relu = relu ? 1 : 0;
  p.res_mode = d->res_mode;
  p.res = res;
  if (d->res_mode && !res) return fail(VT_ERR_INVALID, "residual mode without residual tensor");
  if (d->res_mode == 1 || d->res_mode == 2) {
    const int rT = d->res_mode == 2 ? (p.To + 1) / 2 : p.To;
    set_res(p, cl_strides(rT, p.Ho, p.Wo, p.Co, cw));
    p.resT = rT;
    const bool mix = d->res_mode == 2 || (e && e->res_mix);
    p.ra = mix ? d->alpha : 1.f; p.rb = mix ? 1.f - d->alpha : 1.f;
  } else if (d->res_mode == 3) {
    set_res(p, cl_strides(d->Ti, p.Ho, p.Wo, p.Co, cw));
    p.resT = d->Ti;
    p.ra = d->alpha; p.rb = 1.f - d->alpha;
    if (e) { p.res_t_mode = e->res_t_mode; p.res_cache = e->res_t_mode == 2 ? cache : nullptr; }
  } else {
    p.ra = 0.f; p.rb = 1.f;
  }
  const int taps = d->kt * d->kh * d->kw, K = taps * d->Ci;
  const DType tout = out_f32 ? DT_F32 : ta;
  TcLnFusion lf;
  if (e && e->ln_mode) {
    if (!gamma || !beta || (e->ln_mode == 2 && !out2)) return fail(VT_ERR_INVALID, "fused LayerNorm needs gamma, beta (and out2 for mode 2)");
    if (precision == VT_PREC_FMA32 || force_simt) return fail(VT_ERR_INVALID, "the LayerNorm epilogue exists on the wgmma path only");
    lf.mode = e->ln_mode; lf.silu = e->ln_silu != 0; lf.gamma = gamma; lf.beta = beta; lf.out2 = out2;
  }
  float* wkn = nullptr;
  bf16* wnk = nullptr;
  cudaError_t er;
  const bool want_tc = precision != VT_PREC_FMA32 && !force_simt;
  if (relu && !want_tc) return fail(VT_ERR_INVALID, "the ReLU epilogue exists on the wgmma path only");
  if (want_tc) {
    float wsc = 0.f;
    if (ta == DT_SPLIT) {
      int rc = op_weight_scale(w, (long long)d->Co * K, kModelWeightHeadroom, s, &wsc);
      if (rc) return rc;
      p.acc_scale = 1.0f / wsc;
    }
    TcPlan pl;
    if (!conv_tc_plan(p, tout, &lf, reg, 1, &pl)) return fail(VT_ERR_INVALID, "wgmma conv does not support this geometry: %s", conv_tc_last_error());
    if (pl.ln.mode != lf.mode || (reg && reg->mode && !pl.reg.mode)) return fail(VT_ERR_INVALID, "epilogue cannot be fused: %s", conv_tc_last_error());
    const int Co_pad = (d->Co + 31) / 32 * 32;
    VT_CUDA(cudaMalloc(&wnk, (size_t)K * Co_pad * sizeof(bf16) * cw));
    VT_CUDA(launch_pack_w_nk_bf16(w, wnk, d->Co, Co_pad, d->Ci, taps, K, s, wsc));
    er = launch_conv_tc(pl, (const bf16*)x, wnk, out, s);
  } else {
    VT_CUDA(cudaMalloc(&wkn, (size_t)K * d->Co * sizeof(float)));
    VT_CUDA(launch_pack_w_kn(w, wkn, d->Co, d->Ci, taps, s));
    er = launch_conv_simt(p, ta, tout, ta, x, wkn, out, s);
  }
  cudaError_t e2 = cudaStreamSynchronize(s);
  if (wkn) cudaFree(wkn);
  if (wnk) cudaFree(wnk);
  if (er != cudaSuccess) return fail(VT_ERR_CUDA, "conv launch: %s %s", cudaGetErrorString(er), conv_tc_last_error());
  if (e2 != cudaSuccess) return fail(VT_ERR_CUDA, "conv execution: %s", cudaGetErrorString(e2));
  return VT_OK;
}

int32_t vt_op_conv(int32_t precision, int32_t force_simt, const vt_conv_desc* d, const void* x, const float* w,
                   const float* bias, const void* res, void* out, void* stream) {
  return op_conv_impl(precision, force_simt, d, nullptr, x, nullptr, w, bias, res, nullptr, nullptr, out, nullptr, (cudaStream_t)stream);
}
int32_t vt_op_conv_ex(int32_t precision, const vt_conv_ex* e, const void* x, const void* cache, const float* w,
                      const float* bias, const void* res, const float* gamma, const float* beta, void* out, void* out2,
                      void* stream) {
  if (!e) return fail(VT_ERR_INVALID, "null argument");
  return op_conv_impl(precision, e->force_simt, &e->d, e, x, cache, w, bias, res, gamma, beta, out, out2, (cudaStream_t)stream);
}

// Encoder conv_out with the regularizer in its epilogue, as the model path runs it: x channels-last activation,
// h_out (optional) fp32 [B,Co,T,H,W]; KL: Co = 2*zc, noise/z fp32 [B,zc,T,H,W], kl_loss = 0.5 * sum / B;
// FSQ: Co = zc = number of levels, z = codes, indices int32 [B,T,H,W].  ex carries the geometry and the v1.1 time
// padding (t_mode, cacheT with `cache`); its output fields are ignored (the head output is always fp32 [B,C,T,H,W]).
int32_t vt_op_conv_regularize_ex(int32_t precision, const vt_conv_ex* ex, const void* x, const void* cache, const float* w,
                                 const float* bias, int32_t reg_mode, int32_t zc, const int32_t* fsq_levels, const float* noise,
                                 float* h_out, float* z, int32_t* indices, float* kl_loss, void* stream) {
  if (!ex || !z) return fail(VT_ERR_INVALID, "null argument");
  if (precision != VT_PREC_BF16 && precision != VT_PREC_EXACT_TC) return fail(VT_ERR_INVALID, "the regularizer epilogue exists on the wgmma path only");
  cudaStream_t s = (cudaStream_t)stream;
  const vt_conv_desc* d = &ex->d;
  vt_conv_ex e;
  memset(&e, 0, sizeof(e));
  e.d = *d;
  e.t_mode = ex->t_mode;
  e.cacheT = ex->cacheT;
  e.out_f32_ncdhw = 1;
  TcRegFusion rf;
  rf.mode = reg_mode; rf.zc = zc; rf.z = z; rf.noise = noise; rf.indices = indices; rf.sample = noise ? 1 : 0;
  double* acc = nullptr;
  if (reg_mode == 1) {
    VT_CUDA(cudaMalloc(&acc, sizeof(double)));
    VT_CUDA(launch_kl_clear(acc, s));
    rf.kl_acc = acc;
  } else if (reg_mode == 2) {
    if (!fsq_levels) return fail(VT_ERR_INVALID, "FSQ needs the level list");
    for (int i = 0; i < zc && i < VT_MAX_FSQ; ++i) rf.fsq_levels[i] = fsq_levels[i];
  } else {
    return fail(VT_ERR_INVALID, "reg_mode must be 1 (KL) or 2 (FSQ)");
  }
  int rc = op_conv_impl(precision, 0, d, &e, x, cache, w, bias, nullptr, nullptr, nullptr, h_out, nullptr, s, &rf);
  if (rc == VT_OK && reg_mode == 1 && kl_loss) {
    cudaError_t er = launch_kl_finish(acc, d->B, kl_loss, s);
    if (er == cudaSuccess) er = cudaStreamSynchronize(s);
    if (er != cudaSuccess) rc = fail(VT_ERR_CUDA, "kl finish: %s", cudaGetErrorString(er));
  }
  if (acc) cudaFree(acc);
  return rc;
}
// the same with v1.0 zero time padding
int32_t vt_op_conv_regularize(int32_t precision, const vt_conv_desc* d, const void* x, const float* w, const float* bias,
                              int32_t reg_mode, int32_t zc, const int32_t* fsq_levels, const float* noise, float* h_out,
                              float* z, int32_t* indices, float* kl_loss, void* stream) {
  if (!d) return fail(VT_ERR_INVALID, "null argument");
  vt_conv_ex e;
  memset(&e, 0, sizeof(e));
  e.d = *d;
  return vt_op_conv_regularize_ex(precision, &e, x, nullptr, w, bias, reg_mode, zc, fsq_levels, noise, h_out, z, indices, kl_loss, stream);
}

// Encoder stem (conv_in from the caller's fp32 [B,Ci,T,H,W] tensor) on the conv_stem kernel.
int32_t vt_op_conv_stem(int32_t precision, const float* x, const float* w, const float* bias, void* out, int32_t B,
                        int32_t Ci, int32_t T, int32_t H, int32_t W, int32_t Co, int32_t t_rep, void* stream) {
  if (!x || !w || !out) return fail(VT_ERR_INVALID, "null argument");
  if (precision != VT_PREC_BF16 && precision != VT_PREC_EXACT_TC) return fail(VT_ERR_INVALID, "the stem kernel is a wgmma kernel (BF16 / EXACT_TC)");
  cudaStream_t s = (cudaStream_t)stream;
  const bool split = precision == VT_PREC_EXACT_TC;
  ConvP p = stem_p(B, Ci, T, H, W, Co, t_rep, split, bias);
  if (!conv_stem_supported(p)) return fail(VT_ERR_INVALID, "stem kernel does not take this geometry");
  bf16* wpk = nullptr;
  float wsc = 0.f;
  if (split) {
    int rc = op_weight_scale(w, (long long)Co * Ci * 27, kModelWeightHeadroom, s, &wsc);
    if (rc) return rc;
    p.acc_scale = 1.0f / wsc;
  }
  VT_CUDA(cudaMalloc(&wpk, (size_t)Co * 128 * 2 * sizeof(bf16)));
  VT_CUDA(launch_pack_w_nk_bf16(w, wpk, Co, Co, Ci, 27, 128, s, wsc));
  cudaError_t er = launch_conv_stem(p, x, wpk, (bf16*)out, s);
  cudaError_t e2 = cudaStreamSynchronize(s);
  cudaFree(wpk);
  if (er != cudaSuccess || e2 != cudaSuccess) return fail(VT_ERR_CUDA, "conv_stem: %s", cudaGetErrorString(er != cudaSuccess ? er : e2));
  return VT_OK;
}

// Decoder head (conv_out Cin -> Co <= 4, 3x3x3, v1.0 zero padding, first to_off output frames dropped) as the BF16 path
// runs it: tap-planes GEMM + gather.  x bf16 channels-last [B,T,H,W,Ci]; out fp32 [B,Co,T - to_off,H,W].
int32_t vt_op_head_planes(const void* x, const float* w, const float* bias, float* out, int32_t B, int32_t T, int32_t H,
                          int32_t W, int32_t Ci, int32_t Co, int32_t to_off, void* stream) {
  if (!x || !w || !bias || !out) return fail(VT_ERR_INVALID, "null argument");
  if (Co > 4 || Ci % 64 != 0 || W % 8 != 0) return fail(VT_ERR_INVALID, "head planes need Co <= 4, Cin % 64 == 0, W % 8 == 0");
  cudaStream_t s = (cudaStream_t)stream;
  bf16 *wp = nullptr, *P = nullptr;
  VT_CUDA(cudaMalloc(&wp, (size_t)128 * Ci * sizeof(bf16)));
  VT_CUDA(cudaMalloc(&P, (size_t)B * T * H * W * 128 * sizeof(bf16)));
  VT_CUDA(launch_pack_w_tap_planes(w, wp, Co, Ci, 128, s));
  ConvP p = conv_p(B, T, H, W, Ci);
  set_in(p, cl_strides(T, H, W, Ci, 1));
  p.To = T; p.Ho = H; p.Wo = W; p.Co = 128;
  set_out(p, cl_strides(T, H, W, 128, 1));
  p.kt = p.kh = p.kw = 1;
  p.ra = 0.f; p.rb = 1.f;
  TcPlan pl;
  cudaError_t er = conv_tc_plan(p, DT_BF16, nullptr, nullptr, 1, &pl) ? cudaSuccess : cudaErrorInvalidValue;
  if (er == cudaSuccess) er = launch_conv_tc(pl, (const bf16*)x, wp, P, s);
  if (er == cudaSuccess) er = launch_tap_planes_gather(P, bias, out, B, T, H, W, 128, Co, to_off, s);
  cudaError_t e2 = cudaStreamSynchronize(s);
  cudaFree(wp); cudaFree(P);
  if (er != cudaSuccess || e2 != cudaSuccess) return fail(VT_ERR_CUDA, "head planes: %s %s", cudaGetErrorString(er != cudaSuccess ? er : e2), conv_tc_last_error());
  return VT_OK;
}

// "nearest 2x upsample, then conv" exactly as the tensor-core modes run it: phase-collapsed weights, one small conv per
// output parity class, strided stores into the full-resolution tensor (Exec::up / Exec::time_up), optional fused
// LayerNorm(+SiLU) of the result into out2.
//   kind 0: Upsample (model_3dcausal.py:208-212): x [B,T,H,W,C] -> out [B,T,2H,2W,Co], w [Co,C,3,3]
//   kind 1: TimeUpsampleResCausal2x, v1.0 (:267-273): out [B,2T,H,W,C] = alpha*x' + (1-alpha)*conv(x'), w [C,C,3,3,3]
int32_t vt_op_upsample_conv(int32_t precision, int32_t kind, const void* x, const float* w, const float* bias, float alpha,
                            const float* gamma, const float* beta, int32_t ln_silu, void* out, void* out2, int32_t B,
                            int32_t T, int32_t H, int32_t W, int32_t Ci, int32_t Co, void* stream) {
  if (!x || !w || !bias || !out) return fail(VT_ERR_INVALID, "null argument");
  if (precision != VT_PREC_BF16 && precision != VT_PREC_EXACT_TC) return fail(VT_ERR_INVALID, "phase-collapsed convs exist in the tensor-core modes only");
  if (Ci % 64 != 0 || Co % 32 != 0 || (kind == 1 && Ci != Co)) return fail(VT_ERR_INVALID, "unsupported channel counts");
  cudaStream_t s = (cudaStream_t)stream;
  vt_model dummy;
  memset(&dummy.desc, 0, sizeof(dummy.desc));
  dummy.desc.norm_type = VT_NORM_LAYERNORM;
  dummy.desc.version = 0;
  const bool split = precision == VT_PREC_EXACT_TC;
  const int nph = kind == 0 ? 4 : 2, taps2 = kind == 0 ? 4 : 18;
  bf16* wp = nullptr;
  const size_t per = (size_t)Co * taps2 * Ci;
  VT_CUDA(cudaMalloc(&wp, per * nph * (split ? 2 : 1) * sizeof(bf16)));
  LevelW lv;
  const int id3[3] = {0, 1, 2}, id1[3] = {0, 0, 0};
  const int lo[3] = {0, 1, 1}, hi[3] = {0, 0, 1};
  float wsc = 0.f;
  if (split) {
    int rcw = op_weight_scale(w, (long long)Co * Ci * (kind == 0 ? 9 : 27), kModelWeightHeadroom, s, &wsc);
    if (rcw) { cudaFree(wp); return rcw; }
  }
  lv.resample.Co = Co; lv.resample.Ci = Ci; lv.tconv.Co = Co; lv.tconv.Ci = Ci;
  for (int i = 0; i < nph; ++i) {
    ConvW& ph = kind == 0 ? lv.up_ph[i] : lv.tup_ph[i];
    if (kind == 0) phase_conv(ph, lv.resample, 1, 2, 2);
    else phase_conv(ph, lv.tconv, 2, 3, 3);
    ph.bias = bias;
    if (split) ph.wscale3 = wsc;
    bf16* dst = wp + per * i * (split ? 2 : 1);
    if (split) ph.w_nk3 = dst; else ph.w_nk = dst;
    if (kind == 0) VT_CUDA(launch_pack_w_collapsed(w, dst, Co, Co, Ci, 1, 3, 3, id1, (i >> 1) == 0 ? lo : hi, (i & 1) == 0 ? lo : hi, 1, 2, 2, s, wsc));
    else VT_CUDA(launch_pack_w_collapsed(w, dst, Co, Co, Ci, 3, 3, 3, i == 0 ? hi : lo, id3, id3, 2, 3, 3, s, wsc));
  }
  lv.has_resample = kind == 0; lv.has_up_phase = kind == 0;
  lv.has_tres = kind == 1; lv.has_tup_phase = kind == 1;
  lv.alpha = alpha;
  lv.tkey = "op";
  NormW nw;
  nw.C = Co; nw.gamma = gamma; nw.beta = beta;
  const bool want_ln = gamma && beta && out2;
  const size_t esz = split ? 4 : 2;
  const size_t in_bytes = (size_t)B * T * H * W * Ci * esz;
  const size_t out_elems = kind == 0 ? (size_t)B * T * 4 * H * W * Co : (size_t)B * 2 * T * H * W * Co;
  const size_t ws_bytes = in_bytes + 2 * out_elems * esz + (1 << 20);
  void* ws = nullptr;
  cudaError_t em = cudaMalloc(&ws, ws_bytes);
  if (em != cudaSuccess) { cudaFree(wp); return fail(VT_ERR_CUDA, "cudaMalloc(workspace)"); }
  int rc = VT_OK;
  {
    Exec ex(&dummy, precision, s, ws, ws_bytes, false);
    Exec::Stream st;
    st.x = ex.new_act(B, T, H, W, Ci);
    if (ex.ok()) ex.cuda(cudaMemcpyAsync(st.x.p, x, in_bytes, cudaMemcpyDeviceToDevice, s), "copy in");
    if (kind == 0) ex.up(lv, st, want_ln ? &nw : nullptr, ln_silu != 0);
    else ex.time_up(lv, st, want_ln ? &nw : nullptr, ln_silu != 0);
    if (ex.ok()) ex.cuda(cudaMemcpyAsync(out, st.x.p, out_elems * esz, cudaMemcpyDeviceToDevice, s), "copy out");
    if (ex.ok() && want_ln) {
      if (!st.n.p) ex.rc = fail(VT_ERR_INVALID, "the LayerNorm was not fused into the phase convolutions");
      else ex.cuda(cudaMemcpyAsync(out2, st.n.p, out_elems * esz, cudaMemcpyDeviceToDevice, s), "copy out2");
    }
    rc = ex.rc;
  }
  cudaError_t e2 = cudaStreamSynchronize(s);
  cudaFree(ws); cudaFree(wp);
  if (rc) return rc;
  if (e2 != cudaSuccess) return fail(VT_ERR_CUDA, "upsample conv: %s", cudaGetErrorString(e2));
  return VT_OK;
}

// Fused temporal residual block (BF16, C = 128) exactly as the model path launches it.
static int32_t op_tblock(const void* n1, const void* x, const float* w1, const float* b1, const float* g2, const float* be2,
                         const float* w2, const float* b2, const float* g3, const float* be3, int32_t out_silu, void* out,
                         void* out2, int32_t B, int32_t T, int32_t H, int32_t W, int32_t C, void* stream, const TbCache* cache) {
  if (!n1 || !x || !w1 || !b1 || !g2 || !be2 || !w2 || !b2 || !out) return fail(VT_ERR_INVALID, "null argument");
  if (!tblock_tc_supported(B, T, H, W, C)) return fail(VT_ERR_INVALID, "fused temporal block does not take this geometry: %s", tblock_tc_last_error());
  cudaStream_t s = (cudaStream_t)stream;
  bf16* wp = nullptr;
  const size_t per = (size_t)C * 3 * C;
  VT_CUDA(cudaMalloc(&wp, 2 * per * sizeof(bf16)));
  VT_CUDA(launch_pack_w_nk_bf16(w1, wp, C, C, C, 3, 3 * C, s));
  VT_CUDA(launch_pack_w_nk_bf16(w2, wp + per, C, C, C, 3, 3 * C, s));
  cudaError_t er = launch_tblock_tc((const bf16*)n1, (const bf16*)x, wp, b1, g2, be2, wp + per, b2, (bf16*)out, (bf16*)out2,
                                    out2 ? g3 : nullptr, out2 ? be3 : nullptr, out_silu != 0, B, T, H, W, s, cache);
  cudaError_t e2 = cudaStreamSynchronize(s);
  cudaFree(wp);
  if (er != cudaSuccess || e2 != cudaSuccess) return fail(VT_ERR_CUDA, "tblock: %s %s", cudaGetErrorString(er != cudaSuccess ? er : e2), tblock_tc_last_error());
  return VT_OK;
}
int32_t vt_op_tblock(const void* n1, const void* x, const float* w1, const float* b1, const float* g2, const float* be2,
                     const float* w2, const float* b2, const float* g3, const float* be3, int32_t out_silu, void* out,
                     void* out2, int32_t B, int32_t T, int32_t H, int32_t W, int32_t C, void* stream) {
  return op_tblock(n1, x, w1, b1, g2, be2, w2, b2, g3, be3, out_silu, out, out2, B, T, H, W, C, stream, nullptr);
}
int32_t vt_op_tblock_cached(const void* n1, const void* x, const float* w1, const float* b1, const float* g2, const float* be2,
                            const float* w2, const float* b2, const float* g3, const float* be3, int32_t out_silu, void* out,
                            void* out2, const void* n1_cache_in, const void* h_cache_in, void* n1_cache_out, void* h_cache_out,
                            int32_t B, int32_t T, int32_t H, int32_t W, int32_t C, void* stream) {
  if (!n1_cache_out || !h_cache_out) return fail(VT_ERR_INVALID, "null cache output");
  if (!n1_cache_in != !h_cache_in) return fail(VT_ERR_INVALID, "pass both input caches (a continued video) or neither (its first chunk)");
  TbCache c;
  c.n1_in = (const bf16*)n1_cache_in; c.h_in = (const bf16*)h_cache_in; c.n1_out = (bf16*)n1_cache_out; c.h_out = (bf16*)h_cache_out;
  return op_tblock(n1, x, w1, b1, g2, be2, w2, b2, g3, be3, out_silu, out, out2, B, T, H, W, C, stream, &c);
}

int32_t vt_op_layernorm(int32_t precision, const void* x, const float* gamma, const float* beta, void* y, int64_t rows,
                        int32_t C, int32_t apply_silu, void* stream) {
  VT_CUDA(launch_layernorm(act_type(precision), x, gamma, beta, y, rows, C, apply_silu != 0, precision != VT_PREC_BF16, (cudaStream_t)stream));
  return VT_OK;
}
int32_t vt_op_groupnorm(int32_t precision, const void* x, const float* gamma, const float* beta, void* y, int64_t frames,
                        int64_t ppf, int32_t C, int32_t per_position, int32_t apply_silu, void* workspace,
                        int64_t workspace_bytes, void* stream) {
  if (!per_position && workspace_bytes < (int64_t)(frames * 32 * 2 * sizeof(float))) return fail(VT_ERR_WORKSPACE, "groupnorm stats need %lld bytes", (long long)(frames * 64 * sizeof(float)));
  VT_CUDA(launch_groupnorm(act_type(precision), x, gamma, beta, y, frames, ppf, C, per_position != 0, apply_silu != 0, precision != VT_PREC_BF16,
                           (float*)workspace, (cudaStream_t)stream));
  return VT_OK;
}
// The attention core the model path runs for this precision and shape: wgmma GEMMs (per-frame K / V^T as the B
// operand) when tokens = H * W and C are multiples of 64 in the tensor-core modes, fp32 FMA GEMMs otherwise.  The
// tokens of a frame are its H x W positions, as in the model, so the launches get the model's tile plan.
int32_t vt_op_attention_hw(int32_t precision, const void* q, const void* k, const void* v, void* o, int32_t frames,
                           int32_t H, int32_t W, int32_t C, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!q || !k || !v || !o || !workspace) return fail(VT_ERR_INVALID, "null argument");
  if (precision != VT_PREC_FMA32 && precision != VT_PREC_BF16 && precision != VT_PREC_EXACT_TC)
    return fail(VT_ERR_INVALID, "operator precision must be FMA32, BF16 or EXACT_TC");
  if (frames <= 0 || H <= 0 || W <= 0 || C <= 0) return fail(VT_ERR_INVALID, "attention: empty shape");
  const long long tokens = (long long)H * W;
  vt_model dummy;
  memset(&dummy.desc, 0, sizeof(dummy.desc));
  Exec ex(&dummy, precision, (cudaStream_t)stream, workspace, (size_t)workspace_bytes, false);
  Act aq, ak, av;
  aq.B = frames; aq.T = 1; aq.H = H; aq.W = W; aq.C = C;
  ak = aq; av = aq;
  aq.p = const_cast<void*>(q); ak.p = const_cast<void*>(k); av.p = const_cast<void*>(v);
  Act ao = ex.attention_core(aq, ak, av);
  if (ex.ok()) ex.cuda(cudaMemcpyAsync(o, ao.p, (size_t)frames * tokens * C * dtype_size(ex.ta), cudaMemcpyDeviceToDevice, ex.s), "copy out");
  return ex.rc;
}
// The same for a token count without a frame geometry: the tokens are laid out as an image 8 wide when tokens % 8 == 0
// (one row otherwise), which is not the tile plan of a model frame of H x W (vt_op_attention_hw).
int32_t vt_op_attention(int32_t precision, const void* q, const void* k, const void* v, void* o, int32_t frames,
                        int32_t tokens, int32_t C, void* workspace, int64_t workspace_bytes, void* stream) {
  const bool w8 = tokens > 0 && tokens % 8 == 0;
  return vt_op_attention_hw(precision, q, k, v, o, frames, w8 ? tokens / 8 : 1, w8 ? 8 : tokens, C, workspace, workspace_bytes, stream);
}
// ---- video I/O adjacent steps ---------------------------------------------------------------------------
int32_t vt_video_u8_to_clip(const uint8_t* frames, float* clip, int32_t T, int32_t Hs, int32_t Ws, int32_t C, int32_t h0,
                            int32_t w0, int32_t H, int32_t W, void* stream) {
  if (!frames || !clip) return fail(VT_ERR_INVALID, "null argument");
  if (T <= 0 || C <= 0 || H <= 0 || W <= 0 || h0 < 0 || w0 < 0 || h0 + H > Hs || w0 + W > Ws) return fail(VT_ERR_INVALID, "crop window outside the frame");
  VT_CUDA(launch_u8_frames_to_clip(frames, clip, T, Hs, Ws, C, h0, w0, H, W, (cudaStream_t)stream));
  return VT_OK;
}
int32_t vt_video_u8_to_clip_resized(const uint8_t* frames, float* clip, int32_t N, int32_t Hs, int32_t Ws, int32_t C, int32_t Hr,
                                    int32_t Wr, int32_t h0, int32_t w0, int32_t H, int32_t W, int32_t Tc, void* stream) {
  if (!frames || !clip) return fail(VT_ERR_INVALID, "null argument");
  if (N <= 0 || C <= 0 || Hs <= 0 || Ws <= 0 || Hr <= 0 || Wr <= 0 || Tc <= 0 || N % Tc != 0)
    return fail(VT_ERR_INVALID, "bad shape: N=%d Tc=%d (N must be a positive multiple of Tc)", N, Tc);
  if (H <= 0 || W <= 0 || h0 < 0 || w0 < 0 || h0 + H > Hr || w0 + W > Wr) return fail(VT_ERR_INVALID, "crop window outside the resized frame");
  if (!u8_frames_resize_fits(Hs, Ws, C, Hr, Wr, h0, w0, H, W))
    return fail(VT_ERR_INVALID, "resize %dx%d -> %dx%d: scale too large, the source window of one output pixel does not fit in "
                "shared memory", Hs, Ws, Hr, Wr);
  VT_CUDA(launch_u8_frames_resize_to_clip(frames, clip, N, Hs, Ws, C, Hr, Wr, h0, w0, H, W, Tc, (cudaStream_t)stream));
  return VT_OK;
}
int32_t vt_clip_to_video_u8(const float* clip, uint8_t* frames, int32_t C, int32_t T, int32_t H, int32_t W, void* stream) {
  if (!frames || !clip) return fail(VT_ERR_INVALID, "null argument");
  if (T <= 0 || C <= 0 || H <= 0 || W <= 0) return fail(VT_ERR_INVALID, "bad shape");
  VT_CUDA(launch_clip_to_u8_frames(clip, frames, C, T, H, W, (cudaStream_t)stream));
  return VT_OK;
}

// ---- scoring a reconstruction ---------------------------------------------------------------------------
int64_t vt_frame_scores_workspace_bytes(int32_t B, int32_t C, int32_t T, int32_t H, int32_t W) {
  if (B <= 0 || C <= 0 || T <= 0 || H <= 0 || W <= 0) { fail(VT_ERR_INVALID, "bad shape"); return -1; }
  const long long b = frame_scores_workspace(B, C, T, H, W);
  if (b < 0) fail(VT_ERR_INVALID, "frame scores: %d x %d x %d frames of %d x %d are more tiles than one launch holds; split the batch", B, C, T, H, W);
  return b;
}
int32_t vt_frame_scores(const void* x, int32_t x_dtype, const void* y, int32_t y_dtype, int32_t B, int32_t C, int32_t T, int32_t H,
                        int32_t W, float* psnr, float* ssim, double* running, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!x || !y || !psnr || !workspace) return fail(VT_ERR_INVALID, "null argument");
  if (x_dtype < VT_DTYPE_F32 || x_dtype > VT_DTYPE_F16 || y_dtype < VT_DTYPE_F32 || y_dtype > VT_DTYPE_F16)
    return fail(VT_ERR_INVALID, "unknown dtype (x %d, y %d): VT_DTYPE_F32, VT_DTYPE_BF16 or VT_DTYPE_F16", x_dtype, y_dtype);
  const int64_t need = vt_frame_scores_workspace_bytes(B, C, T, H, W);
  if (need < 0) return VT_ERR_INVALID;
  if (ssim && !frame_scores_has_ssim(H, W)) {
    const int f = frame_scores_pool_factor(H, W);
    return fail(VT_ERR_INVALID, "SSIM kernel size can't be greater than actual input size. Input size: %d x %d (%d x %d pooled by %d). "
                "Kernel size: 11 x 11", H / f, W / f, H, W, f);
  }
  if (workspace_bytes < need) return fail(VT_ERR_WORKSPACE, "workspace too small for the frame scores: %lld < %lld bytes", (long long)workspace_bytes, (long long)need);
  VT_CUDA(launch_frame_scores(x, x_dtype, y, y_dtype, B, C, T, H, W, psnr, ssim, running, workspace, (cudaStream_t)stream));
  return VT_OK;
}

int32_t vt_op_fsq(const float* h, int32_t d, const int32_t* levels, int64_t P, int32_t B, float* codes, int32_t* indices,
                  void* stream) {
  VT_CUDA(launch_fsq(h, d, levels, P, B, codes, indices, (cudaStream_t)stream));
  return VT_OK;
}
int32_t vt_op_fsq_indices_to_codes(const int32_t* indices, int32_t d, const int32_t* levels, int64_t P, int32_t B,
                                   float* codes, void* stream) {
  VT_CUDA(launch_fsq_indices_to_codes(indices, d, levels, P, B, codes, (cudaStream_t)stream));
  return VT_OK;
}
int64_t vt_fsq_aux_workspace_bytes(int32_t d, const int32_t* levels, int64_t tokens) {
  if (!levels) { fail(VT_ERR_INVALID, "null argument"); return -1; }
  FsqAuxGeom g;
  const char* why = fsq_aux_geometry(d, levels, tokens, &g);
  if (why) { fail(VT_ERR_INVALID, "%s", why); return -1; }
  return (int64_t)fsq_aux_workspace(g);
}
int32_t vt_fsq_aux_partials(const float* h, int32_t d, const int32_t* levels, int64_t P, int32_t B, float inv_temperature,
                            float* stats, float* avg_prob, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h || !levels || !stats || !avg_prob || !workspace) return fail(VT_ERR_INVALID, "null argument");
  if (B <= 0 || P <= 0) return fail(VT_ERR_INVALID, "bad shape");
  FsqAuxGeom g;
  const char* why = fsq_aux_geometry(d, levels, (long long)B * P, &g);
  if (why) return fail(VT_ERR_INVALID, "%s", why);
  if ((size_t)workspace_bytes < fsq_aux_workspace(g)) return fail(VT_ERR_WORKSPACE, "workspace too small for the FSQ aux loss");
  VT_CUDA(launch_fsq_aux_partials(h, g, levels, P, inv_temperature, stats, avg_prob, workspace, (cudaStream_t)stream));
  return VT_OK;
}
int32_t vt_fsq_aux_finalize(const float* stats, const float* avg_prob, int32_t n_segments, int32_t d, const int32_t* levels,
                            int32_t world_size, float entropy_weight, float diversity_gamma, float commitment_weight,
                            float* aux_loss, float* components, void* stream) {
  if (!stats || !avg_prob || !levels || !aux_loss) return fail(VT_ERR_INVALID, "null argument");
  if (n_segments <= 0 || world_size <= 0) return fail(VT_ERR_INVALID, "n_segments and world_size must be positive");
  FsqAuxGeom g;
  const char* why = fsq_aux_geometry(d, levels, 1, &g);
  if (why) return fail(VT_ERR_INVALID, "%s", why);
  VT_CUDA(launch_fsq_aux_finalize(stats, avg_prob, n_segments, g.J, world_size, entropy_weight, diversity_gamma, commitment_weight,
                                  aux_loss, components, (cudaStream_t)stream));
  return VT_OK;
}
int32_t vt_op_kl(const float* h, const float* noise, int32_t zc, int64_t P, int32_t B, int32_t sample, float* z,
                 float* kl_loss, void* stream) {
  double* scratch = nullptr;
  VT_CUDA(cudaMalloc(&scratch, sizeof(double)));
  cudaError_t e = launch_kl(h, noise, zc, P, B, sample != 0, z, kl_loss, scratch, (cudaStream_t)stream);
  cudaStreamSynchronize((cudaStream_t)stream);
  cudaFree(scratch);
  if (e != cudaSuccess) return fail(VT_ERR_CUDA, "kl: %s", cudaGetErrorString(e));
  return VT_OK;
}


// ---- LPIPS (vidtok/modules/lpips.py; scripts/inference_evaluate.py:175-186) --------------------------------------------
// VGG16 features[0:30] as 13 ReLU convolutions (conv1_1 on the LPIPS stem, the rest on conv_tc), four 2x2 max-pools, and the
// head of each of the five taps, walked over the frame pairs in passes of at most lpips_pass_frames() pairs.  Image f < g of a
// pass is frame n0 + f of x, image g + f the same frame of y, so each layer runs both images in one launch.
}  // extern "C"
namespace {
struct LpipsConv { int Ci, Co, pw, pb; };
// the reference's state-dict indices of the 13 convolutions, their slices and channels; taps after conv 1, 3, 6, 9, 12, a
// max-pool in front of conv 2, 4, 7, 10
constexpr int kLpConvIdx[13] = {0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28};
constexpr int kLpSlice[13] = {1, 1, 2, 2, 3, 3, 3, 4, 4, 4, 5, 5, 5};
constexpr int kLpCo[13] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
constexpr int kLpChns[5] = {64, 128, 256, 512, 512};
inline bool lp_tap(int i) { return i == 1 || i == 3 || i == 6 || i == 9 || i == 12; }
inline bool lp_pool_before(int i) { return i == 2 || i == 4 || i == 7 || i == 10; }
// 2^31: the kernels are not audited for activations of more elements (DESIGN.md section 6)
constexpr long long kLpMaxElems = 1LL << 31;
}  // namespace

struct vt_lpips_model {
  int device = 0;
  std::vector<vt::Param> params;
  std::map<std::string, int> index;
  float* pool = nullptr;
  int64_t pool_elems = 0;
  bool finalized = false;
  vt::bf16* packed = nullptr;          // every conv's bf16 [Co][Kpad], then its split copy [Co][hi Kpad | lo Kpad]
  LpipsConv conv[13];
  vt::bf16* w[13] = {nullptr};
  vt::bf16* w3[13] = {nullptr};
  float wscale3[13] = {0.f};
  int plin[5] = {0};
};

extern "C" {

// frame pairs of one pass: 16, or fewer where relu1_2 of the pass (2 g images x H x W x 64) would exceed 2^31 elements;
// 0 when not even one pair fits
static int lpips_pass_frames(int H, int W) {
  const long long per = 2LL * H * W * 64;
  int g = 16;
  while (g > 0 && g * per > kLpMaxElems) --g;
  return g;
}
// the spatial extents of the five levels (floor halving)
static void lpips_levels(int H, int W, int (&Hl)[5], int (&Wl)[5]) {
  Hl[0] = H; Wl[0] = W;
  for (int l = 1; l < 5; ++l) { Hl[l] = Hl[l - 1] / 2; Wl[l] = Wl[l - 1] / 2; }
}
struct LpipsLayout {
  int G, Hl[5], Wl[5];
  size_t act_bytes, part_bytes;
};
static int lpips_check(int precision, int B, int C, int T, int H, int W, LpipsLayout* L) {
  if (precision != VT_PREC_BF16 && precision != VT_PREC_EXACT_TC) return fail(VT_ERR_INVALID, "LPIPS runs in BF16 or EXACT_TC, got precision %d", precision);
  if (C != 3) return fail(VT_ERR_INVALID, "LPIPS takes RGB clips (C == 3), got C = %d", C);
  if (B <= 0 || T <= 0) return fail(VT_ERR_INVALID, "empty clip (B = %d, T = %d)", B, T);
  if (H < 16 || W < 16) return fail(VT_ERR_INVALID, "frames of %d x %d are smaller than 16 x 16, where relu5_3 is 1 x 1", H, W);
  const int Gmax = lpips_pass_frames(H, W);
  if (Gmax < 1) return fail(VT_ERR_INVALID, "frames of %d x %d give activations beyond 2^31 elements", H, W);
  const long long frames = (long long)B * T;
  L->G = (int)(frames < Gmax ? frames : Gmax);
  lpips_levels(H, W, L->Hl, L->Wl);
  const size_t esz = precision == VT_PREC_EXACT_TC ? 4 : 2;
  L->act_bytes = align_up((size_t)2 * L->G * H * W * 64 * esz, 1024);
  long long tiles = 0;
  for (int k = 0; k < 5; ++k) tiles += lpips_head_tiles(L->Hl[k], L->Wl[k]);
  L->part_bytes = align_up((size_t)L->G * tiles * sizeof(float), 1024);
  return VT_OK;
}

// The conv_tc plan of conv i (i >= 1) for a pass of g pairs at level extent H x W
static bool lpips_conv_plan(const vt_lpips_model* h, int i, int g, int H, int W, bool split, TcPlan* pl) {
  const LpipsConv& c = h->conv[i];
  const long long cw = split ? 2 : 1;
  ConvP p = conv_p(2 * g, 1, H, W, c.Ci);
  p.split = split ? 1 : 0;
  set_in(p, cl_strides(1, H, W, c.Ci, cw));
  p.kt = 1; p.kh = p.kw = 3; p.ph = p.pw = 1;
  p.Co = c.Co;
  conv_out_size(p, 0, 1, 1);
  set_out(p, cl_strides(1, p.Ho, p.Wo, c.Co, cw));
  p.bias = h->finalized ? h->pool + h->params[c.pb].offset : nullptr;
  p.ra = 0.f; p.rb = 1.f;
  p.relu = 1;
  p.acc_scale = split ? 1.0f / h->wscale3[i] : 0.f;
  return conv_tc_plan(p, split ? DT_SPLIT : DT_BF16, nullptr, nullptr, 1, pl);
}

int32_t vt_lpips_create(int32_t device, vt_lpips_model** out) {
  if (!out) return fail(VT_ERR_INVALID, "null argument");
  vt_lpips_model* h = new vt_lpips_model();
  h->device = device;
  auto add = [&](const std::string& name, std::vector<int64_t> shape) {
    Param p;
    p.name = name;
    p.shape = shape;
    p.numel = 1;
    for (auto d : shape) p.numel *= d;
    p.offset = h->pool_elems;
    h->pool_elems += (p.numel + 3) / 4 * 4;
    h->index[name] = (int)h->params.size();
    h->params.push_back(p);
    return (int)h->params.size() - 1;
  };
  int Ci = 3;
  for (int i = 0; i < 13; ++i) {
    const std::string key = "net.slice" + std::to_string(kLpSlice[i]) + "." + std::to_string(kLpConvIdx[i]);
    h->conv[i].Ci = Ci;
    h->conv[i].Co = kLpCo[i];
    h->conv[i].pw = add(key + ".weight", {kLpCo[i], Ci, 3, 3});
    h->conv[i].pb = add(key + ".bias", {kLpCo[i]});
    Ci = kLpCo[i];
  }
  for (int k = 0; k < 5; ++k) h->plin[k] = add("lin" + std::to_string(k) + ".model.1.weight", {1, kLpChns[k], 1, 1});
  *out = h;
  return VT_OK;
}

void vt_lpips_destroy(vt_lpips_model* h) {
  if (!h) return;
  if (h->pool) cudaFree(h->pool);
  if (h->packed) cudaFree(h->packed);
  delete h;
}

int32_t vt_lpips_num_params(const vt_lpips_model* h) { return h ? (int32_t)h->params.size() : 0; }

int32_t vt_lpips_param_info(const vt_lpips_model* h, int32_t i, char* name, int32_t cap, int64_t* shape4, int32_t* ndim) {
  if (!h || i < 0 || i >= (int)h->params.size()) return fail(VT_ERR_INVALID, "bad parameter index");
  const Param& p = h->params[i];
  if (name && cap > 0) {
    strncpy(name, p.name.c_str(), cap - 1);
    name[cap - 1] = 0;
  }
  if (ndim) *ndim = (int)p.shape.size();
  if (shape4)
    for (size_t k = 0; k < 4; ++k) shape4[k] = k < p.shape.size() ? p.shape[k] : 1;
  return VT_OK;
}

static int lpips_device(vt_lpips_model* h) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    return fail(VT_ERR_NO_DEVICE, "no CUDA device visible: vidtok_b200 has no CPU fallback");
  }
  VT_CUDA(cudaSetDevice(h->device));
  if (!h->pool) VT_CUDA(cudaMalloc(&h->pool, (size_t)h->pool_elems * sizeof(float)));
  return VT_OK;
}

int32_t vt_lpips_load_param(vt_lpips_model* h, const char* name, const float* data, int64_t numel, int32_t is_device, void* stream) {
  if (!h || !name || !data) return fail(VT_ERR_INVALID, "null argument");
  auto it = h->index.find(name);
  if (it == h->index.end()) return fail(VT_ERR_INVALID, "unknown LPIPS parameter %s", name);
  Param& p = h->params[it->second];
  if (p.numel != numel) return fail(VT_ERR_INVALID, "parameter %s: expected %lld elements, got %lld", name, (long long)p.numel, (long long)numel);
  int rc = lpips_device(h);
  if (rc) return rc;
  VT_CUDA(cudaMemcpyAsync(h->pool + p.offset, data, (size_t)numel * sizeof(float), is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                          (cudaStream_t)stream));
  p.loaded = true;
  h->finalized = false;
  return VT_OK;
}

// Repacks the convolutions' weights: bf16 [Co][K = tap * Ci + ci] (conv1_1: K padded to 128 for the stem) and the split copy
// of w * 2^s, s from max |w| of each convolution.
int32_t vt_lpips_finalize(vt_lpips_model* h, void* stream) {
  if (!h) return fail(VT_ERR_INVALID, "null argument");
  for (auto& p : h->params)
    if (!p.loaded) return fail(VT_ERR_NOT_READY, "LPIPS parameter %s was never loaded", p.name.c_str());
  int rc = lpips_device(h);
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  auto kpad = [&](int i) { return i == 0 ? 128 : 9 * h->conv[i].Ci; };
  size_t total = 0;
  for (int i = 0; i < 13; ++i) total += 3 * align_up((size_t)h->conv[i].Co * kpad(i), 512);
  if (!h->packed) VT_CUDA(cudaMalloc(&h->packed, total * sizeof(bf16)));
  {
    float* d_max = nullptr;
    VT_CUDA(cudaMalloc(&d_max, 13 * sizeof(float)));
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 13 && e == cudaSuccess; ++i)
      e = launch_absmax(h->pool + h->params[h->conv[i].pw].offset, (long long)h->conv[i].Co * h->conv[i].Ci * 9, d_max + i, s);
    float h_max[13];
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_max, d_max, sizeof(h_max), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    cudaFree(d_max);
    if (e != cudaSuccess) return fail(VT_ERR_CUDA, "LPIPS weight scales: %s", cudaGetErrorString(e));
    for (int i = 0; i < 13; ++i) h->wscale3[i] = split_weight_scale(h_max[i]);
  }
  size_t off = 0;
  for (int i = 0; i < 13; ++i) {
    const LpipsConv& c = h->conv[i];
    const size_t n = align_up((size_t)c.Co * kpad(i), 512);
    h->w[i] = h->packed + off;
    h->w3[i] = h->packed + off + n;
    off += 3 * n;
    const float* w = h->pool + h->params[c.pw].offset;
    VT_CUDA(launch_pack_w_nk_bf16(w, h->w[i], c.Co, c.Co, c.Ci, 9, kpad(i), s));
    VT_CUDA(launch_pack_w_nk_bf16(w, h->w3[i], c.Co, c.Co, c.Ci, 9, kpad(i), s, h->wscale3[i]));
  }
  VT_CUDA(cudaStreamSynchronize(s));
  h->finalized = true;
  return VT_OK;
}

int32_t vt_lpips_pass_frames(int32_t H, int32_t W) { return H > 0 && W > 0 ? lpips_pass_frames(H, W) : 0; }

int64_t vt_lpips_workspace_bytes(const vt_lpips_model* h, int32_t precision, int32_t B, int32_t C, int32_t T, int32_t H, int32_t W) {
  if (!h) { fail(VT_ERR_INVALID, "null handle"); return -1; }
  LpipsLayout L;
  if (lpips_check(precision, B, C, T, H, W, &L)) return -1;
  return (int64_t)(2 * L.act_bytes + L.part_bytes);
}

int32_t vt_lpips(vt_lpips_model* h, int32_t precision, const void* x, int32_t x_dtype, const void* y, int32_t y_dtype, int32_t B, int32_t C,
                 int32_t T, int32_t H, int32_t W, float* lpips, float* per_layer, double* running, void* workspace, int64_t workspace_bytes,
                 void* stream) {
  if (!h || !x || !y || !lpips) return fail(VT_ERR_INVALID, "null argument");
  auto dt_ok = [](int d) { return d == VT_DTYPE_F32 || d == VT_DTYPE_BF16 || d == VT_DTYPE_F16; };
  if (!dt_ok(x_dtype) || !dt_ok(y_dtype)) return fail(VT_ERR_INVALID, "unknown dtype (x %d, y %d)", x_dtype, y_dtype);
  LpipsLayout L;
  int rc = lpips_check(precision, B, C, T, H, W, &L);
  if (rc) return rc;
  if (!workspace || workspace_bytes < (int64_t)(2 * L.act_bytes + L.part_bytes))
    return fail(VT_ERR_WORKSPACE, "LPIPS workspace: %lld bytes given, %lld needed", (long long)workspace_bytes,
                (long long)(2 * L.act_bytes + L.part_bytes));
  if (!h->finalized) return fail(VT_ERR_NOT_READY, "vt_lpips_finalize has not been called");
  const bool split = precision == VT_PREC_EXACT_TC;
  const long long frames = (long long)B * T;
  // every plan of both pass sizes first: a geometry conv_tc refuses launches nothing
  const int g_tail = (int)(frames % L.G == 0 ? L.G : frames % L.G);
  for (int g : {L.G, g_tail}) {
    int lvl = 0;
    for (int i = 1; i < 13; ++i) {
      if (lp_pool_before(i)) ++lvl;
      TcPlan pl;
      if (!lpips_conv_plan(h, i, g, L.Hl[lvl], L.Wl[lvl], split, &pl))
        return fail(VT_ERR_INVALID, "LPIPS conv %d at %d x %d: the wgmma conv does not take it: %s", kLpConvIdx[i], L.Hl[lvl], L.Wl[lvl],
                    conv_tc_last_error());
    }
  }
  cudaStream_t s = (cudaStream_t)stream;
  bf16* buf[2] = {(bf16*)workspace, (bf16*)((char*)workspace + L.act_bytes)};
  float* part = (float*)((char*)workspace + 2 * L.act_bytes);
  for (long long n0 = 0; n0 < frames; n0 += L.G) {
    const int g = (int)std::min<long long>(L.G, frames - n0);
    LpipsFinish fin;
    long long off = 0;
    for (int k = 0; k < 5; ++k) {
      fin.tiles[k] = lpips_head_tiles(L.Hl[k], L.Wl[k]);
      fin.off[k] = off;
      fin.area[k] = (double)L.Hl[k] * L.Wl[k];
      off += (long long)g * fin.tiles[k];
    }
    int cur = 0, lvl = 0, tap = 0;
    VT_CUDA(launch_lpips_stem(x, x_dtype, y, y_dtype, T, n0, g, H, W, split, split ? h->w3[0] : h->w[0], h->pool + h->params[h->conv[0].pb].offset,
                              1.0f / h->wscale3[0], buf[cur], s));
    for (int i = 1; i < 13; ++i) {
      if (lp_pool_before(i)) {
        VT_CUDA(launch_maxpool2x2(buf[cur], buf[cur ^ 1], 2LL * g, L.Hl[lvl], L.Wl[lvl], h->conv[i].Ci, split, s));
        cur ^= 1;
        ++lvl;
      }
      TcPlan pl;
      lpips_conv_plan(h, i, g, L.Hl[lvl], L.Wl[lvl], split, &pl);
      cudaError_t e = launch_conv_tc(pl, buf[cur], split ? h->w3[i] : h->w[i], buf[cur ^ 1], s);
      if (e != cudaSuccess) return fail(VT_ERR_CUDA, "LPIPS conv %d: %s %s", kLpConvIdx[i], cudaGetErrorString(e), conv_tc_last_error());
      cur ^= 1;
      if (lp_tap(i)) {
        VT_CUDA(launch_lpips_head(buf[cur], g, L.Hl[lvl], L.Wl[lvl], h->conv[i].Co, split, h->pool + h->params[h->plin[tap]].offset,
                                  part + fin.off[tap], s));
        ++tap;
      }
    }
    VT_CUDA(launch_lpips_finish(part, fin, g, lpips + n0, per_layer ? per_layer + n0 * 5 : nullptr, running, s));
  }
  return VT_OK;
}

// One ReLU convolution of the LPIPS stack as the executor runs it (vt_conv_desc with res_mode 0)
int32_t vt_op_conv_relu(int32_t precision, const vt_conv_desc* d, const void* x, const float* w, const float* bias, void* out, void* stream) {
  if (!d) return fail(VT_ERR_INVALID, "null argument");
  if (d->res_mode != 0) return fail(VT_ERR_INVALID, "vt_op_conv_relu takes no residual (res_mode 0)");
  if (precision != VT_PREC_BF16 && precision != VT_PREC_EXACT_TC) return fail(VT_ERR_INVALID, "the ReLU epilogue exists on the wgmma path only");
  return op_conv_impl(precision, 0, d, nullptr, x, nullptr, w, bias, nullptr, nullptr, nullptr, out, nullptr, (cudaStream_t)stream,
                      nullptr, true);
}

int32_t vt_op_maxpool2x2(int32_t precision, const void* x, void* y, int64_t N, int32_t H, int32_t W, int32_t C, void* stream) {
  if (!x || !y) return fail(VT_ERR_INVALID, "null argument");
  if (precision != VT_PREC_BF16 && precision != VT_PREC_EXACT_TC) return fail(VT_ERR_INVALID, "maxpool2x2 takes bf16 or split activations");
  if (N <= 0 || H < 2 || W < 2 || C <= 0 || C % 8 != 0) return fail(VT_ERR_INVALID, "maxpool2x2 needs N > 0, H, W >= 2 and C %% 8 == 0");
  VT_CUDA(launch_maxpool2x2((const bf16*)x, (bf16*)y, N, H, W, C, precision == VT_PREC_EXACT_TC, (cudaStream_t)stream));
  return VT_OK;
}

}  // extern "C"
