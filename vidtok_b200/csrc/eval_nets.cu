// Host side of the evaluation networks: LPIPS (VGG16) and I3D for FVD.  Their parameter tables, handles and executors over
// the kernels of lpips.cu, i3d.cu and conv_tc, and the LPIPS operator entry points the tests compare against the reference.
#include "model.h"

#include <algorithm>
#include <cmath>
#include <cstring>

using namespace vt;

// ---- LPIPS (vidtok/modules/lpips.py; scripts/inference_evaluate.py:175-186) --------------------------------------------
// VGG16 features[0:30] as 13 ReLU convolutions (conv1_1 on the LPIPS stem, the rest on conv_tc), four 2x2 max-pools, and the
// head of each of the five taps, walked over the frame pairs in passes of at most lpips_pass_frames() pairs.  Image f < g of a
// pass is frame n0 + f of x, image g + f the same frame of y, so each layer runs both images in one launch.
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
  vt::ParamSet params{"LPIPS "};
  float* pool = nullptr;
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
  const float* bias = h->finalized ? h->pool + h->params[c.pb].offset : nullptr;
  return relu_conv_plan(2 * g, 1, H, W, c.Ci, 1, 3, 0, 0, 1, 1, c.Co, c.Co, bias, h->wscale3[i], split, pl);
}

int32_t vt_lpips_create(int32_t device, vt_lpips_model** out) {
  if (!out) return fail(VT_ERR_INVALID, "null argument");
  vt_lpips_model* h = new vt_lpips_model();
  h->device = device;
  int Ci = 3;
  for (int i = 0; i < 13; ++i) {
    const std::string key = "net.slice" + std::to_string(kLpSlice[i]) + "." + std::to_string(kLpConvIdx[i]);
    h->conv[i].Ci = Ci;
    h->conv[i].Co = kLpCo[i];
    h->conv[i].pw = h->params.add(key + ".weight", {kLpCo[i], Ci, 3, 3});
    h->conv[i].pb = h->params.add(key + ".bias", {kLpCo[i]});
    Ci = kLpCo[i];
  }
  for (int k = 0; k < 5; ++k) h->plin[k] = h->params.add("lin" + std::to_string(k) + ".model.1.weight", {1, kLpChns[k], 1, 1});
  *out = h;
  return VT_OK;
}

void vt_lpips_destroy(vt_lpips_model* h) {
  if (!h) return;
  if (h->pool) cudaFree(h->pool);
  if (h->packed) cudaFree(h->packed);
  delete h;
}

int32_t vt_lpips_num_params(const vt_lpips_model* h) { return h ? h->params.size() : 0; }

int32_t vt_lpips_param_info(const vt_lpips_model* h, int32_t i, char* name, int32_t cap, int64_t* shape4, int32_t* ndim) {
  return h ? h->params.info(i, name, cap, shape4, 4, ndim) : fail(VT_ERR_INVALID, "bad parameter index");
}

static int lpips_device(vt_lpips_model* h) {
  int rc = use_device(h->device);
  if (rc) return rc;
  if (!h->pool) VT_CUDA(cudaMalloc(&h->pool, (size_t)h->params.pool_elems * sizeof(float)));
  return VT_OK;
}

int32_t vt_lpips_load_param(vt_lpips_model* h, const char* name, const float* data, int64_t numel, int32_t is_device, void* stream) {
  if (!h || !name || !data) return fail(VT_ERR_INVALID, "null argument");
  const int i = h->params.find(name, numel);
  if (i < 0) return VT_ERR_INVALID;
  int rc = lpips_device(h);
  if (rc) return rc;
  VT_CUDA(cudaMemcpyAsync(h->pool + h->params[i].offset, data, (size_t)numel * sizeof(float), is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                          (cudaStream_t)stream));
  h->params[i].loaded = true;
  h->finalized = false;
  return VT_OK;
}

// Repacks the convolutions' weights: bf16 [Co][K = tap * Ci + ci] (conv1_1: K padded to 128 for the stem) and the split copy
// of w * 2^s, s from max |w| of each convolution.
int32_t vt_lpips_finalize(vt_lpips_model* h, void* stream) {
  if (!h) return fail(VT_ERR_INVALID, "null argument");
  int rc = h->params.check_loaded();
  if (!rc) rc = lpips_device(h);
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  auto kpad = [&](int i) { return i == 0 ? 128 : 9 * h->conv[i].Ci; };
  size_t total = 0;
  for (int i = 0; i < 13; ++i) total += 3 * align_up((size_t)h->conv[i].Co * kpad(i), 512);
  if (!h->packed) VT_CUDA(cudaMalloc(&h->packed, total * sizeof(bf16)));
  std::vector<std::pair<const float*, long long>> ws;
  for (const LpipsConv& c : h->conv) ws.push_back({h->pool + h->params[c.pw].offset, (long long)c.Co * c.Ci * 9});
  rc = split_weight_scales(ws, 1.0f, s, h->wscale3);
  if (rc) return rc;
  size_t off = 0;
  for (int i = 0; i < 13; ++i) {
    const LpipsConv& c = h->conv[i];
    const size_t n = align_up((size_t)c.Co * kpad(i), 512);
    h->w[i] = h->packed + off;
    h->w3[i] = h->packed + off + n;
    off += 3 * n;
    const float* w = h->pool + h->params[c.pw].offset;
    VT_CUDA(pack_conv_weights(w, h->w[i], h->w3[i], c.Co, c.Co, c.Ci, 9, kpad(i), h->wscale3[i], s));
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


// ---- I3D features for FVD (metrics.py: the Frechet video distance) ----------------------------------------------------------
// Inception-v1 inflated, Kinetics-400, in the parameter layout of the PyTorch port (InceptionI3d): every unit is a bias-free
// convolution, BatchNorm3d (eps 1e-3, folded into the packed weights and a bias at finalize) and ReLU, with "SAME" zero
// padding.  Conv3d_1a_7x7 runs on i3d_stem_kernel from the resized clip, the 56 other units on conv_tc with the ReLU epilogue,
// the max-pools on maxpool3d_kernel, the head on i3d_head_kernel.  Branch widths are stored in zero-padded channel slices
// (outputs to multiples of 32, every tensor a later conv reads to a multiple of 64); each branch of an Inception module
// writes its slice of the module's output directly through the output strides.  Clips run in passes of
// i3d_pass_clips(T) clips; a clip's features do not depend on the pass or the call.
}  // extern "C"
namespace {
struct I3dConv {
  std::string key;
  int Ci = 0, Co = 0, k = 1;    // real channels, k x k x k taps
  int Ci_s = 0, Co_s = 0;       // channels of the stored input tensor; channels this conv writes (rows >= Co are zero)
  I3dSegs in;                   // where the real input channels sit in the stored input
  int pw = -1, pg = -1, pb = -1, pm = -1, pv = -1;
  bf16* w = nullptr;            // [Co_s][Kpad] bf16
  bf16* w3 = nullptr;           // split copy of w * wscale3
  float* bias = nullptr;        // [Co_s], BatchNorm folded, zero beyond Co
  float wscale3 = 1.f;
  int kpad() const { return Ci_s == 3 ? 1088 : k * k * k * Ci_s; }
};
// the Inception modules' branch widths [o0 .. o5]: b0 1x1 -> o0; b1a 1x1 -> o1, b1b 3x3x3 -> o2; b2a 1x1 -> o3, b2b 3x3x3 ->
// o4; b3a max-pool 3x3x3, b3b 1x1 -> o5; output [b0, b1b, b2b, b3b]
constexpr int kI3dMods[9][6] = {{64, 96, 128, 16, 32, 32},     {128, 128, 192, 32, 96, 64},   {192, 96, 208, 16, 48, 64},
                                {160, 112, 224, 24, 64, 64},   {128, 128, 256, 24, 64, 64},   {112, 144, 288, 32, 64, 64},
                                {256, 160, 320, 32, 128, 128}, {256, 160, 320, 32, 128, 128}, {384, 192, 384, 48, 128, 128}};
const char* const kI3dModNames[9] = {"Mixed_3b", "Mixed_3c", "Mixed_4b", "Mixed_4c", "Mixed_4d", "Mixed_4e", "Mixed_4f", "Mixed_5b", "Mixed_5c"};
struct I3dModule {
  int conv[6];                  // b0, b1a, b1b, b2a, b2b, b3b
  int Cout_s;
  I3dSegs out;                  // the four branch slices of the output
};
// the end points in network order: 0 stem, 1 unit, 2 max-pool, 3 module (idx: conv or module index)
struct I3dStep { int kind, idx, k[3], s[3]; const char* name; };
const I3dStep kI3dSteps[16] = {
    {0, 0, {7, 7, 7}, {2, 2, 2}, "Conv3d_1a_7x7"},  {2, -1, {1, 3, 3}, {1, 2, 2}, "MaxPool3d_2a_3x3"},
    {1, 1, {1, 1, 1}, {1, 1, 1}, "Conv3d_2b_1x1"},  {1, 2, {3, 3, 3}, {1, 1, 1}, "Conv3d_2c_3x3"},
    {2, -1, {1, 3, 3}, {1, 2, 2}, "MaxPool3d_3a_3x3"}, {3, 0, {}, {}, "Mixed_3b"}, {3, 1, {}, {}, "Mixed_3c"},
    {2, -1, {3, 3, 3}, {2, 2, 2}, "MaxPool3d_4a_3x3"}, {3, 2, {}, {}, "Mixed_4b"}, {3, 3, {}, {}, "Mixed_4c"},
    {3, 4, {}, {}, "Mixed_4d"}, {3, 5, {}, {}, "Mixed_4e"}, {3, 6, {}, {}, "Mixed_4f"},
    {2, -1, {2, 2, 2}, {2, 2, 2}, "MaxPool3d_5a_2x2"}, {3, 7, {}, {}, "Mixed_5b"}, {3, 8, {}, {}, "Mixed_5c"}};
constexpr int kI3dSteps_n = 16;
inline int up32(int c) { return (c + 31) / 32 * 32; }
inline int up64(int c) { return (c + 63) / 64 * 64; }
inline I3dSegs seg_identity(int c) {
  I3dSegs s;
  memset(&s, 0, sizeof(s));
  s.n = 1; s.real = c; s.count[0] = c;
  return s;
}
inline int seg_map(const I3dSegs& s, int c) {
  for (int k = 0; k < s.n; ++k)
    if (c >= s.real0[k] && c < s.real0[k] + s.count[k]) return s.stored0[k] + c - s.real0[k];
  return -1;
}
// "SAME" padding of one axis: front padding and output extent
inline void i3d_same(int n, int k, int s, int& front, int& out) {
  const int pad = n % s == 0 ? std::max(k - s, 0) : std::max(k - n % s, 0);
  front = pad / 2;
  out = (n + s - 1) / s;
}
// an activation: extent and stored channel layout
struct I3dAct {
  int T, H, W, Cs;
  I3dSegs segs;
};
// 2^31: the kernels are not audited for activations of more elements (DESIGN.md section 6), as kLpMaxElems
constexpr long long kI3dMaxElems = 1LL << 31;
constexpr int kI3dMaxPass = 8;
}  // namespace

struct vt_i3d_model {
  int device = 0;
  vt::ParamSet params{"I3D "};
  std::vector<std::vector<float>> host;   // the loaded parameters (finalize folds and packs them)
  bool finalized = false;
  std::vector<I3dConv> conv;               // 0 stem, 1 Conv3d_2b, 2 Conv3d_2c, then six per module
  I3dModule mod[9];
  int plw = -1, plb = -1;
  std::vector<void*> allocs;
  float* lw = nullptr;                     // logits weights transposed, [1024][400] fp32
  float* lb = nullptr;                     // [400]
};

extern "C" {

// The activations of one clip at every end point (stored channels), and the largest of each workspace role
struct I3dGeom {
  I3dAct act[kI3dSteps_n];
  long long trunk = 0, t1 = 0, t2 = 0, pool = 0;   // elements per clip
};
static void i3d_geometry(const vt_i3d_model* h, int T, I3dGeom* g) {
  I3dAct a{T, kI3dSize, kI3dSize, 3, seg_identity(3)};
  *g = I3dGeom();
  auto pos = [](const I3dAct& x) { return (long long)x.T * x.H * x.W; };
  for (int i = 0; i < kI3dSteps_n; ++i) {
    const I3dStep& st = kI3dSteps[i];
    if (st.kind == 0 || st.kind == 2) {
      int f, To, Ho, Wo;
      i3d_same(a.T, st.k[0], st.s[0], f, To);
      i3d_same(a.H, st.k[1], st.s[1], f, Ho);
      i3d_same(a.W, st.k[2], st.s[2], f, Wo);
      a.T = To; a.H = Ho; a.W = Wo;
      if (st.kind == 0) { a.Cs = 64; a.segs = seg_identity(64); }
    } else if (st.kind == 1) {
      a.Cs = h->conv[st.idx].Co_s;
      a.segs = seg_identity(h->conv[st.idx].Co);
    } else {
      const I3dModule& m = h->mod[st.idx];
      g->t1 = std::max(g->t1, pos(a) * h->conv[m.conv[1]].Co_s);
      g->t2 = std::max(g->t2, pos(a) * h->conv[m.conv[3]].Co_s);
      g->pool = std::max(g->pool, pos(a) * a.Cs);
      a.Cs = m.Cout_s;
      a.segs = m.out;
    }
    g->act[i] = a;
    g->trunk = std::max(g->trunk, pos(a) * a.Cs);
  }
}

// clips per pass: 8, or fewer where the resized clips or an activation of the pass would exceed 2^31 elements; 0 for T < 9
static int i3d_pass_clips(const vt_i3d_model* h, int T) {
  if (T < 9) return 0;
  I3dGeom g;
  i3d_geometry(h, T, &g);
  const long long per = std::max({3LL * T * kI3dSize * kI3dSize, g.trunk, g.t1, g.t2, g.pool});
  int n = kI3dMaxPass;
  while (n > 0 && n * per > kI3dMaxElems) --n;
  return n;
}

struct I3dLayout {
  int G;
  I3dGeom geom;
  size_t prep, trunk, t1, t2, pool, total;
};
static int i3d_check(const vt_i3d_model* h, int precision, int B, int C, int T, int H, int W, I3dLayout* L) {
  if (precision != VT_PREC_BF16 && precision != VT_PREC_EXACT_TC) return fail(VT_ERR_INVALID, "I3D runs in BF16 or EXACT_TC, got precision %d", precision);
  if (C != 3) return fail(VT_ERR_INVALID, "I3D takes RGB clips (C == 3), got C = %d", C);
  if (B <= 0 || H <= 0 || W <= 0) return fail(VT_ERR_INVALID, "empty clip (B = %d, H = %d, W = %d)", B, H, W);
  if (T < 9) return fail(VT_ERR_INVALID, "I3D needs clips of at least 9 frames (2 time steps at Mixed_5c for the [2,7,7] pool), got T = %d", T);
  const int Gmax = i3d_pass_clips(h, T);
  if (Gmax < 1) return fail(VT_ERR_INVALID, "clips of %d frames give I3D activations beyond 2^31 elements", T);
  L->G = B < Gmax ? B : Gmax;
  i3d_geometry(h, T, &L->geom);
  const size_t esz = precision == VT_PREC_EXACT_TC ? 4 : 2;
  L->prep = align_up((size_t)L->G * 3 * T * kI3dSize * kI3dSize * 4, 1024);
  L->trunk = align_up((size_t)L->G * L->geom.trunk * esz, 1024);
  L->t1 = align_up((size_t)L->G * L->geom.t1 * esz, 1024);
  L->t2 = align_up((size_t)L->G * L->geom.t2 * esz, 1024);
  L->pool = align_up((size_t)L->G * L->geom.pool * esz, 1024);
  L->total = L->prep + 2 * L->trunk + L->t1 + L->t2 + L->pool;
  return VT_OK;
}

// The conv_tc plan of a stride-1 unit over a pass of G clips, writing channels [c0, c0 + Co_s) of an output with out_Cs
// channels (the caller offsets the output pointer by c0)
static bool i3d_unit_plan(const I3dConv& c, int G, const I3dAct& in, int out_Cs, bool split, TcPlan* pl) {
  const int front = (c.k - 1) / 2, back = c.k - 1 - front;
  return relu_conv_plan(G, in.T, in.H, in.W, c.Ci_s, c.k, c.k, front, back, front, back, c.Co_s, out_Cs, c.bias, c.wscale3, split, pl);
}

// every conv_tc plan of a pass of G clips, before anything is launched
static int i3d_plan_all(const vt_i3d_model* h, int G, const I3dLayout& L, bool split) {
  TcPlan pl;
  for (int i = 0; i < kI3dSteps_n; ++i) {
    const I3dStep& st = kI3dSteps[i];
    const I3dAct& in = L.geom.act[i - 1 < 0 ? 0 : i - 1];
    auto check = [&](const I3dConv& c, const I3dAct& a, int out_Cs) -> int {
      if (!i3d_unit_plan(c, G, a, out_Cs, split, &pl))
        return fail(VT_ERR_INVALID, "I3D %s at %dx%dx%d: the wgmma conv does not take it: %s", c.key.c_str(), a.T, a.H, a.W, conv_tc_last_error());
      return VT_OK;
    };
    int rc = VT_OK;
    if (st.kind == 1) rc = check(h->conv[st.idx], in, h->conv[st.idx].Co_s);
    if (st.kind == 3) {
      const I3dModule& m = h->mod[st.idx];
      const int Cout = m.Cout_s;
      I3dAct a1 = in, a2 = in, ap = in;
      a1.Cs = h->conv[m.conv[1]].Co_s;
      a2.Cs = h->conv[m.conv[3]].Co_s;
      for (int r : {0, 1, 3}) if (!rc) rc = check(h->conv[m.conv[r]], in, r == 0 ? Cout : h->conv[m.conv[r]].Co_s);
      if (!rc) rc = check(h->conv[m.conv[2]], a1, Cout);
      if (!rc) rc = check(h->conv[m.conv[4]], a2, Cout);
      if (!rc) rc = check(h->conv[m.conv[5]], ap, Cout);
    }
    if (rc) return rc;
  }
  return VT_OK;
}

static int i3d_unit(const vt_i3d_model* h, const I3dConv& c, int G, const I3dAct& in, const bf16* x, bf16* out, int out_Cs, bool split,
                    cudaStream_t s) {
  TcPlan pl;
  if (!i3d_unit_plan(c, G, in, out_Cs, split, &pl)) return fail(VT_ERR_INVALID, "I3D %s: %s", c.key.c_str(), conv_tc_last_error());
  const cudaError_t e = launch_conv_tc(pl, x, split ? c.w3 : c.w, out, s);
  if (e != cudaSuccess) return fail(VT_ERR_CUDA, "I3D %s: %s %s", c.key.c_str(), cudaGetErrorString(e), conv_tc_last_error());
  return VT_OK;
}
static int i3d_pool(const I3dAct& in, const I3dAct& out, const int (&k)[3], const int (&st)[3], int G, const bf16* x, bf16* y, bool split,
                    cudaStream_t s) {
  MaxPool3d q;
  int o;
  q.T = in.T; q.H = in.H; q.W = in.W; q.C = in.Cs;
  q.kt = k[0]; q.kh = k[1]; q.kw = k[2]; q.st = st[0]; q.sh = st[1]; q.sw = st[2];
  i3d_same(in.T, k[0], st[0], q.pt, o);
  i3d_same(in.H, k[1], st[1], q.ph, o);
  i3d_same(in.W, k[2], st[2], q.pw, o);
  q.To = out.T; q.Ho = out.H; q.Wo = out.W;
  VT_CUDA(launch_maxpool3d(x, y, G, q, split, s));
  return VT_OK;
}

// One pass of G clips (clips [n0, n0 + G) of x) up to and including end point `last`; *res = the trunk buffer holding it
static int i3d_pass(const vt_i3d_model* h, bool split, const void* x, int x_dtype, long long n0, int G, int T, int H, int W,
                    const I3dLayout& L, char* ws, int last, bf16** res, cudaStream_t s) {
  float* prep = (float*)ws;
  bf16* buf[2] = {(bf16*)(ws + L.prep), (bf16*)(ws + L.prep + L.trunk)};
  bf16* t1 = (bf16*)(ws + L.prep + 2 * L.trunk);
  bf16* t2 = (bf16*)(ws + L.prep + 2 * L.trunk + L.t1);
  bf16* pp = (bf16*)(ws + L.prep + 2 * L.trunk + L.t1 + L.t2);
  VT_CUDA(launch_i3d_resize(x, x_dtype, n0, G, T, H, W, prep, s));
  int cur = 0, rc = VT_OK;
  for (int i = 0; i <= last && !rc; ++i) {
    const I3dStep& st = kI3dSteps[i];
    const I3dAct& out = L.geom.act[i];
    if (st.kind == 0) {
      const I3dConv& c = h->conv[0];
      int pt, ph, pw, o;
      i3d_same(T, 7, 2, pt, o);
      i3d_same(kI3dSize, 7, 2, ph, o);
      i3d_same(kI3dSize, 7, 2, pw, o);
      VT_CUDA(launch_i3d_stem(prep, G, T, out.T, pt, ph, pw, split, split ? c.w3 : c.w, c.bias, 1.0f / c.wscale3, buf[cur], s));
      continue;
    }
    const I3dAct& in = L.geom.act[i - 1];
    if (st.kind == 1) {
      rc = i3d_unit(h, h->conv[st.idx], G, in, buf[cur], buf[cur ^ 1], out.Cs, split, s);
    } else if (st.kind == 2) {
      rc = i3d_pool(in, out, st.k, st.s, G, buf[cur], buf[cur ^ 1], split, s);
    } else {
      const I3dModule& m = h->mod[st.idx];
      const bf16* X = buf[cur];
      bf16* Y = buf[cur ^ 1];
      I3dAct a1 = in, a2 = in;
      a1.Cs = h->conv[m.conv[1]].Co_s;
      a2.Cs = h->conv[m.conv[3]].Co_s;
      const int k3[3] = {3, 3, 3}, s1[3] = {1, 1, 1};
      if (!rc) rc = i3d_unit(h, h->conv[m.conv[0]], G, in, X, Y + m.out.stored0[0], m.Cout_s, split, s);
      if (!rc) rc = i3d_unit(h, h->conv[m.conv[1]], G, in, X, t1, a1.Cs, split, s);
      if (!rc) rc = i3d_unit(h, h->conv[m.conv[2]], G, a1, t1, Y + m.out.stored0[1], m.Cout_s, split, s);
      if (!rc) rc = i3d_unit(h, h->conv[m.conv[3]], G, in, X, t2, a2.Cs, split, s);
      if (!rc) rc = i3d_unit(h, h->conv[m.conv[4]], G, a2, t2, Y + m.out.stored0[2], m.Cout_s, split, s);
      if (!rc) rc = i3d_pool(in, in, k3, s1, G, X, pp, split, s);
      if (!rc) rc = i3d_unit(h, h->conv[m.conv[5]], G, in, pp, Y + m.out.stored0[3], m.Cout_s, split, s);
    }
    cur ^= 1;
  }
  *res = buf[cur];
  return rc;
}

int32_t vt_i3d_create(int32_t device, vt_i3d_model** out) {
  if (!out) return fail(VT_ERR_INVALID, "null argument");
  vt_i3d_model* h = new vt_i3d_model();
  h->device = device;
  auto unit = [&](const std::string& key, int Ci, int Co, int k, int Ci_s, const I3dSegs& in, int Co_s) {
    I3dConv c;
    c.key = key; c.Ci = Ci; c.Co = Co; c.k = k; c.Ci_s = Ci_s; c.in = in; c.Co_s = Co_s;
    c.pw = h->params.add(key + ".conv3d.weight", {Co, Ci, k, k, k});
    c.pg = h->params.add(key + ".bn.weight", {Co});
    c.pb = h->params.add(key + ".bn.bias", {Co});
    c.pm = h->params.add(key + ".bn.running_mean", {Co});
    c.pv = h->params.add(key + ".bn.running_var", {Co});
    h->conv.push_back(c);
    return (int)h->conv.size() - 1;
  };
  unit("Conv3d_1a_7x7", 3, 64, 7, 3, seg_identity(3), 64);
  unit("Conv3d_2b_1x1", 64, 64, 1, 64, seg_identity(64), 64);
  unit("Conv3d_2c_3x3", 64, 192, 3, 64, seg_identity(64), 192);
  int Cin = 192, Cin_s = 192;
  I3dSegs in = seg_identity(192);
  for (int m = 0; m < 9; ++m) {
    const int* o = kI3dMods[m];
    const std::string key = kI3dModNames[m];
    I3dModule& M = h->mod[m];
    int w[4] = {up32(o[0]), up32(o[2]), up32(o[4]), up32(o[5])};
    const int tot = w[0] + w[1] + w[2] + w[3];
    w[3] += up64(tot) - tot;   // the last slice takes the padding up to a multiple of 64 channels
    M.Cout_s = up64(tot);
    memset(&M.out, 0, sizeof(M.out));
    M.out.n = 4;
    const int real[4] = {o[0], o[2], o[4], o[5]};
    for (int b = 0, r = 0, sidx = 0; b < 4; ++b) {
      M.out.real0[b] = r; M.out.stored0[b] = sidx; M.out.count[b] = real[b];
      r += real[b]; sidx += w[b];
    }
    M.out.real = o[0] + o[2] + o[4] + o[5];
    M.conv[0] = unit(key + ".b0", Cin, o[0], 1, Cin_s, in, w[0]);
    M.conv[1] = unit(key + ".b1a", Cin, o[1], 1, Cin_s, in, up64(o[1]));
    M.conv[2] = unit(key + ".b1b", o[1], o[2], 3, up64(o[1]), seg_identity(o[1]), w[1]);
    M.conv[3] = unit(key + ".b2a", Cin, o[3], 1, Cin_s, in, up64(o[3]));
    M.conv[4] = unit(key + ".b2b", o[3], o[4], 3, up64(o[3]), seg_identity(o[3]), w[2]);
    M.conv[5] = unit(key + ".b3b", Cin, o[5], 1, Cin_s, in, w[3]);
    Cin = M.out.real; Cin_s = M.Cout_s; in = M.out;
  }
  h->plw = h->params.add("logits.conv3d.weight", {kI3dClasses, kI3dFeatC, 1, 1, 1});
  h->plb = h->params.add("logits.conv3d.bias", {kI3dClasses});
  h->host.resize(h->params.size());
  *out = h;
  return VT_OK;
}

void vt_i3d_destroy(vt_i3d_model* h) {
  if (!h) return;
  for (void* p : h->allocs) cudaFree(p);
  delete h;
}

int32_t vt_i3d_num_params(const vt_i3d_model* h) { return h ? h->params.size() : 0; }

int32_t vt_i3d_param_info(const vt_i3d_model* h, int32_t i, char* name, int32_t cap, int64_t* shape5, int32_t* ndim) {
  return h ? h->params.info(i, name, cap, shape5, 5, ndim) : fail(VT_ERR_INVALID, "bad parameter index");
}

int32_t vt_i3d_load_param(vt_i3d_model* h, const char* name, const float* data, int64_t numel, int32_t is_device, void* stream) {
  if (!h || !name || !data) return fail(VT_ERR_INVALID, "null argument");
  const int i = h->params.find(name, numel);
  if (i < 0) return VT_ERR_INVALID;
  std::vector<float>& v = h->host[i];
  v.resize((size_t)numel);
  if (is_device) {
    VT_CUDA(cudaSetDevice(h->device));
    VT_CUDA(cudaMemcpyAsync(v.data(), data, (size_t)numel * sizeof(float), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    VT_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  } else {
    memcpy(v.data(), data, (size_t)numel * sizeof(float));
  }
  h->params[i].loaded = true;
  h->finalized = false;
  return VT_OK;
}

// Folds each unit's BatchNorm into its weights and a bias (in double, rounded once to fp32), scatters the input channels into
// the stored layout, packs bf16 [Co_s][Kpad] and the split copy of w * 2^s; the logits weights are kept transposed in fp32.
int32_t vt_i3d_finalize(vt_i3d_model* h, void* stream) {
  if (!h) return fail(VT_ERR_INVALID, "null argument");
  int rc = h->params.check_loaded();
  if (!rc) rc = use_device(h->device);
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  VT_CUDA(cudaStreamSynchronize(s));
  for (void* p : h->allocs) cudaFree(p);
  h->allocs.clear();
  auto dev_alloc = [&](size_t bytes, void** p) -> cudaError_t {
    cudaError_t e = cudaMalloc(p, bytes);
    if (e == cudaSuccess) h->allocs.push_back(*p);
    return e;
  };
  size_t max_w = 0;
  for (const I3dConv& c : h->conv) max_w = std::max(max_w, (size_t)c.Co_s * c.Ci_s * c.k * c.k * c.k);
  float* tmp = nullptr;
  VT_CUDA(cudaMalloc(&tmp, max_w * sizeof(float)));
  std::vector<float> wp(max_w), bp;
  for (I3dConv& c : h->conv) {
    const int taps = c.k * c.k * c.k;
    const std::vector<float>& w = h->host[c.pw];
    const std::vector<float>& gm = h->host[c.pg];
    const std::vector<float>& bt = h->host[c.pb];
    const std::vector<float>& mu = h->host[c.pm];
    const std::vector<float>& var = h->host[c.pv];
    std::fill(wp.begin(), wp.begin() + (size_t)c.Co_s * c.Ci_s * taps, 0.f);
    bp.assign(c.Co_s, 0.f);
    float maxabs = 0.f;
    for (int o = 0; o < c.Co; ++o) {
      const double sc = (double)gm[o] / std::sqrt((double)var[o] + 1e-3);
      bp[o] = (float)((double)bt[o] - (double)mu[o] * sc);
      for (int ci = 0; ci < c.Ci; ++ci) {
        const int cs = seg_map(c.in, ci);
        for (int t = 0; t < taps; ++t) {
          const float v = (float)((double)w[((size_t)o * c.Ci + ci) * taps + t] * sc);
          wp[((size_t)o * c.Ci_s + cs) * taps + t] = v;
          maxabs = std::max(maxabs, std::fabs(v));
        }
      }
    }
    c.wscale3 = split_weight_scale(maxabs);
    const size_t nw = align_up((size_t)c.Co_s * c.kpad(), 512);
    cudaError_t e = dev_alloc(3 * nw * sizeof(bf16), (void**)&c.w);
    if (e == cudaSuccess) e = dev_alloc(align_up((size_t)c.Co_s, 64) * sizeof(float), (void**)&c.bias);
    if (e == cudaSuccess) e = cudaMemcpy(tmp, wp.data(), (size_t)c.Co_s * c.Ci_s * taps * sizeof(float), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(c.bias, bp.data(), (size_t)c.Co_s * sizeof(float), cudaMemcpyHostToDevice);
    c.w3 = c.w + nw;
    if (e == cudaSuccess) e = pack_conv_weights(tmp, c.w, c.w3, c.Co_s, c.Co_s, c.Ci_s, taps, c.kpad(), c.wscale3, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);   // tmp is refilled for the next conv
    if (e != cudaSuccess) { rc = fail(VT_ERR_CUDA, "I3D finalize %s: %s", c.key.c_str(), cudaGetErrorString(e)); break; }
  }
  cudaFree(tmp);
  if (rc) return rc;
  std::vector<float> wt((size_t)kI3dFeatC * kI3dClasses);
  for (int o = 0; o < kI3dClasses; ++o)
    for (int c = 0; c < kI3dFeatC; ++c) wt[(size_t)c * kI3dClasses + o] = h->host[h->plw][(size_t)o * kI3dFeatC + c];
  VT_CUDA(dev_alloc(wt.size() * sizeof(float), (void**)&h->lw));
  VT_CUDA(dev_alloc(kI3dClasses * sizeof(float), (void**)&h->lb));
  VT_CUDA(cudaMemcpy(h->lw, wt.data(), wt.size() * sizeof(float), cudaMemcpyHostToDevice));
  VT_CUDA(cudaMemcpy(h->lb, h->host[h->plb].data(), kI3dClasses * sizeof(float), cudaMemcpyHostToDevice));
  h->finalized = true;
  return VT_OK;
}

int32_t vt_i3d_pass_clips(const vt_i3d_model* h, int32_t T, int32_t H, int32_t W) {
  return h && H > 0 && W > 0 ? i3d_pass_clips(h, T) : 0;
}

int64_t vt_i3d_workspace_bytes(const vt_i3d_model* h, int32_t precision, int32_t B, int32_t C, int32_t T, int32_t H, int32_t W) {
  if (!h) { fail(VT_ERR_INVALID, "null handle"); return -1; }
  I3dLayout L;
  if (i3d_check(h, precision, B, C, T, H, W, &L)) return -1;
  return (int64_t)L.total;
}

static int i3d_args(vt_i3d_model* h, int precision, const void* x, int x_dtype, int B, int C, int T, int H, int W, void* workspace,
                    int64_t workspace_bytes, I3dLayout* L) {
  if (!h || !x) return fail(VT_ERR_INVALID, "null argument");
  if (x_dtype != VT_DTYPE_F32 && x_dtype != VT_DTYPE_BF16 && x_dtype != VT_DTYPE_F16) return fail(VT_ERR_INVALID, "unknown dtype %d", x_dtype);
  int rc = i3d_check(h, precision, B, C, T, H, W, L);
  if (rc) return rc;
  if (!workspace || workspace_bytes < (int64_t)L->total)
    return fail(VT_ERR_WORKSPACE, "I3D workspace: %lld bytes given, %lld needed", (long long)workspace_bytes, (long long)L->total);
  if (!h->finalized) return fail(VT_ERR_NOT_READY, "vt_i3d_finalize has not been called");
  const long long clips = B;
  const int g_tail = (int)(clips % L->G == 0 ? L->G : clips % L->G);
  for (int g : {L->G, g_tail}) {
    rc = i3d_plan_all(h, g, *L, precision == VT_PREC_EXACT_TC);
    if (rc) return rc;
  }
  return VT_OK;
}

int32_t vt_i3d_features(vt_i3d_model* h, int32_t precision, const void* x, int32_t x_dtype, int32_t B, int32_t C, int32_t T, int32_t H, int32_t W,
                        float* features, double* stats, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!features) return fail(VT_ERR_INVALID, "null argument");
  I3dLayout L;
  int rc = i3d_args(h, precision, x, x_dtype, B, C, T, H, W, workspace, workspace_bytes, &L);
  if (rc) return rc;
  const bool split = precision == VT_PREC_EXACT_TC;
  cudaStream_t s = (cudaStream_t)stream;
  for (long long n0 = 0; n0 < B; n0 += L.G) {
    const int g = (int)std::min<long long>(L.G, B - n0);
    bf16* f = nullptr;
    rc = i3d_pass(h, split, x, x_dtype, n0, g, T, H, W, L, (char*)workspace, kI3dSteps_n - 1, &f, s);
    if (rc) return rc;
    VT_CUDA(launch_i3d_head(f, g, L.geom.act[kI3dSteps_n - 1].T, split, h->lw, h->lb, features + n0 * kI3dClasses, s));
    if (stats) VT_CUDA(launch_i3d_stats(features + n0 * kI3dClasses, g, stats, s));
  }
  return VT_OK;
}

int32_t vt_i3d_endpoint(vt_i3d_model* h, int32_t precision, const void* x, int32_t x_dtype, int32_t B, int32_t C, int32_t T, int32_t H,
                        int32_t W, const char* name, float* out, int64_t* shape5, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h || !name) return fail(VT_ERR_INVALID, "null argument");
  int step = -1;
  for (int i = 0; i < kI3dSteps_n; ++i)
    if (!strcmp(name, kI3dSteps[i].name)) step = i;
  if (step < 0) return fail(VT_ERR_INVALID, "unknown I3D end point %s", name);
  I3dLayout L;
  if (!out) {
    int rc = i3d_check(h, precision, B, C, T, H, W, &L);
    if (rc) return rc;
  } else {
    int rc = i3d_args(h, precision, x, x_dtype, B, C, T, H, W, workspace, workspace_bytes, &L);
    if (rc) return rc;
    if (B > L.G) return fail(VT_ERR_INVALID, "vt_i3d_endpoint runs one pass: at most %d clips at T = %d, got %d", L.G, T, B);
  }
  const I3dAct& a = L.geom.act[step];
  if (shape5) {
    shape5[0] = B; shape5[1] = a.segs.real; shape5[2] = a.T; shape5[3] = a.H; shape5[4] = a.W;
  }
  if (!out) return VT_OK;
  const bool split = precision == VT_PREC_EXACT_TC;
  cudaStream_t s = (cudaStream_t)stream;
  bf16* f = nullptr;
  int rc = i3d_pass(h, split, x, x_dtype, 0, B, T, H, W, L, (char*)workspace, step, &f, s);
  if (rc) return rc;
  VT_CUDA(launch_i3d_unpack(f, split, B, a.T, a.H, a.W, a.Cs, a.segs, out, s));
  return VT_OK;
}

}  // extern "C"
