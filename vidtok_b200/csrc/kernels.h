// Host-callable launchers of the vidtok_b200 kernels (internal; the public surface is include/vidtok_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace vt {

// DT_SPLIT: fp32-class activations stored as two fp16 planes side by side in the channel dimension,
// [..., hi(C) | lo(C)] with hi = fp16(v), lo = fp16(v - hi) (common.cuh: split_store; the operand format of the EXACT_TC mode).
// One logical element = 4 bytes; pointers to such tensors are bf16*, strides in ConvP count bf16 elements.
enum DType { DT_F32 = 0, DT_BF16 = 1, DT_SPLIT = 2 };
inline size_t dtype_size(DType t) { return t == DT_BF16 ? 2 : 4; }

void prof_start();
void prof_set_detail(bool on);
int prof_stop(char* buf, int cap);

// conv_simt.cu
cudaError_t launch_conv_simt(const ConvP& p, DType tin, DType tout, DType tres, const void* x, const float* w_kn,
                             void* out, cudaStream_t s);
cudaError_t launch_gemm_simt(DType ta, DType tb, DType tc, const void* A, const void* B, void* C, int M, int N, int K,
                             long long lda, long long sbn, long long sbk, long long ldc, int batch, long long bsA,
                             long long bsB, long long bsC, float scale, cudaStream_t s);

// elementwise.cu
cudaError_t launch_layernorm(DType t, const void* x, const float* gamma, const float* beta, void* y, long long rows,
                             int C, bool silu, bool exact, cudaStream_t s);
// Element counts / strides of the data-movement launchers (upsample_nearest, cache_update, copy_frames) are LOGICAL
// elements; a DT_SPLIT element is moved as one 4-byte unit (whole rows keep their hi|lo layout).
// stats: float2 [frames*32] scratch (per-frame mode)
cudaError_t launch_groupnorm(DType t, const void* x, const float* gamma, const float* beta, void* y, long long frames,
                             long long pos_per_frame, int C, bool per_position, bool silu, bool exact, float* stats,
                             cudaStream_t s);
cudaError_t launch_softmax_rows(DType tout, const float* S, void* P, long long rows, int N, cudaStream_t s);
cudaError_t launch_kl(const float* h, const float* noise, int zc, long long P, int B, bool sample, float* z,
                      float* kl_loss, double* scratch, cudaStream_t s);
cudaError_t launch_fsq(const float* h, int d, const int* levels_host, long long P, int B, float* codes, int* indices,
                       cudaStream_t s);
cudaError_t launch_fsq_indices_to_codes(const int* indices, int d, const int* levels_host, long long P, int B,
                                        float* codes, cudaStream_t s);
// fsq_aux.cu: the FSQ auxiliary loss (regularizers.py:232-245) from the per-channel softmax factors.  One segment (an
// untiled batch or one chunk of a tiled video) gives partials stats [2] = (per_sample_entropy, commit_loss) and
// avg_prob [J]; the finish step combines n segments (avg_prob summed over `world` ranks by the caller, then divided here).
#define VT_FSQ_AUX_MAX_CODEBOOK (1LL << 22)
#define VT_FSQ_AUX_MAX_SUM_LEVELS 256
struct FsqAuxGeom {
  int d = 0, a = 0;                            // digits; the low group is digits [0, a)
  int L[VT_MAX_FSQ] = {0}, off[VT_MAX_FSQ] = {0};   // levels; offset of channel i's table in a token's factor row
  int SL = 0;                                  // sum of the levels (factor row length)
  int J = 0, Jlo = 0, Jhi = 0;                 // codebook = Jlo * Jhi, code j = j_lo + Jlo * j_hi
  int ksplit = 1;                              // token slices of the avg_prob contraction
  long long N = 0, kchunk = 0;                 // tokens; tokens per slice
};
// nullptr, or why the level list / token count is not supported
const char* fsq_aux_geometry(int d, const int* levels, long long N, FsqAuxGeom* g);
size_t fsq_aux_workspace(const FsqAuxGeom& g);
// h fp32 [B, d, P] (tokens n = b * P + p); stats / avg_prob device outputs of this segment
cudaError_t launch_fsq_aux_partials(const float* h, const FsqAuxGeom& g, const int* levels, long long P, float inv_t, float* stats,
                                    float* avg_prob, void* ws, cudaStream_t s);
cudaError_t launch_fsq_aux_finalize(const float* stats, const float* avg_prob, int nseg, int J, int world, float w_ent, float gamma,
                                    float w_commit, float* aux, float* comp, cudaStream_t s);
// weight repacking: w [Co][Ci][taps] (reference OIDHW flattened) -> [K = tap*Ci + ci][Co] fp32
cudaError_t launch_pack_w_kn(const float* w, float* out, int Co, int Ci, int taps, cudaStream_t s);
// -> [Co][K = tap*Ci + ci] bf16 (K-major rows for the wgmma B operand)
// wscale != 0: split rows [hi(Kpad) | lo(Kpad)] (fp16 planes, DT_SPLIT operand format) of w * wscale (see split_weight_scale)
cudaError_t launch_pack_w_nk_bf16(const float* w, bf16* out, int Co, int Co_pad, int Ci, int taps, int Kpad, cudaStream_t s,
                                  float wscale = 0.f);
cudaError_t launch_absmax(const float* w, long long n, float* out, cudaStream_t s);
// Power-of-two scale for the split (fp16 hi|lo) copy of a weight tensor with the given max |w|: largest 2^s with
// 2^s * maxabs * headroom < 4096 (headroom: phase-collapsed weights sum up to 4 taps), so that values at 1e-4 of the maximum
// still have a normal fp16 lo plane.  The conv epilogue multiplies the accumulator by 1 / scale.
inline float split_weight_scale(float maxabs, float headroom = 1.0f) {
  if (!(maxabs > 0.f)) return 1.0f;
  float sc = 1.0f;
  while (sc * maxabs * headroom < 2048.0f && sc < 1.0e30f) sc *= 2.0f;
  while (sc * maxabs * headroom >= 4096.0f && sc > 1.0e-30f) sc *= 0.5f;
  return sc;
}
// The headroom the model uses for every convolution (a phase-collapsed tap sums up to 4 original taps).  The single-operator
// entry points use it too, so that they pick the same scale, and with it the same residual path (res_mma needs 2^s <= 2^15),
// as the model does for the same weights.
constexpr float kModelWeightHeadroom = 4.0f;
// phase-collapsed weights of "nearest-2x upsample then conv": original taps (a,b,c) of a kt x kh x kw kernel are
// summed into tap (mt[a], mh[b], mw[c]) of a kt2 x kh2 x kw2 kernel; output [Co_pad][kt2*kh2*kw2*Ci] bf16
cudaError_t launch_pack_w_collapsed(const float* w, bf16* out, int Co, int Co_pad, int Ci, int kt, int kh, int kw,
                                    const int* mt, const int* mh, const int* mw, int kt2, int kh2, int kw2, cudaStream_t s,
                                    float wscale = 0.f);
// trilinear (align_corners=False) 2x upsampling along T of channels-last x [B,T,HWC] -> [B,2T,HWC]
cudaError_t launch_time_interp2x(DType t, const void* x, void* y, int B, int T, long long hw, int C, cudaStream_t s);
cudaError_t launch_upsample_nearest(DType t, const void* x, void* y, int B, int T, int H, int W, int C, int ut, int uh,
                                    int uw, cudaStream_t s);
cudaError_t launch_cache_update(DType t, const void* x, const void* old_cache, void* new_cache, int B, int Tc, int P,
                                int off, bool first, long long frame_elems, long long x_bs, cudaStream_t s);
cudaError_t launch_ncdhw_to_cl(DType t, const float* x, void* y, int B, int C, int T, int H, int W, int t_rep,
                               cudaStream_t s);
cudaError_t launch_copy_frames(DType t, const void* src, void* dst, int B, long long src_bs, long long dst_bs,
                               long long n_per_batch, cudaStream_t s);
// byte copies of n segments in one launch (vt_chunk_state_copy_slots): segs is a DEVICE table; max_bytes is the largest
// segment, total_bytes the sum (the profiler's byte count)
struct SlotSeg {
  const void* src;
  void* dst;
  unsigned long long bytes;
};
cudaError_t launch_slot_copy(const SlotSeg* segs, int n, unsigned long long max_bytes, unsigned long long total_bytes,
                             cudaStream_t s);

// video I/O adjacent steps: decoded uint8 frames [T,Hs,Ws,C] -> cropped normalised clip fp32 [C,T,H,W]; clip -> uint8 frames
cudaError_t launch_u8_frames_to_clip(const uint8_t* src, float* dst, int T, int Hs, int Ws, int C, int h0, int w0, int H, int W,
                                    cudaStream_t s);
cudaError_t launch_clip_to_u8_frames(const float* src, uint8_t* dst, int C, int T, int H, int W, cudaStream_t s);
// video_io.cu: uint8 frames [N,Hs,Ws,C] -> antialiased bilinear resize to Hr x Wr -> crop (h0,w0,H,W) -> Normalize(.5,.5)
// -> clips fp32 [N/Tc,C,Tc,H,W].  _fits is false when the source window of one output pixel exceeds shared memory (the
// launcher then returns cudaErrorInvalidValue).
bool u8_frames_resize_fits(int Hs, int Ws, int C, int Hr, int Wr, int h0, int w0, int H, int W);
cudaError_t launch_u8_frames_resize_to_clip(const uint8_t* src, float* dst, int N, int Hs, int Ws, int C, int Hr, int Wr, int h0,
                                            int w0, int H, int W, int Tc, cudaStream_t s);
// metrics.cu: per-frame PSNR and SSIM of y against x, both [B,C,T,H,W] in [-1,1] before the clamp (dtype 0 fp32, 1 bf16,
// 2 fp16 = VT_DTYPE_*).  psnr / ssim fp32 [B*T] (ssim may be null: PSNR only); running (may be null) double [3] receives
// += (sum of PSNR, sum of SSIM, frames).  ws: frame_scores_workspace bytes (-1: more tiles than one grid holds).
int frame_scores_pool_factor(int H, int W);   // max(1, round(min(H, W) / 256)), half to even
bool frame_scores_has_ssim(int H, int W);     // the pooled frame holds at least one 11 x 11 window
long long frame_scores_workspace(int B, int C, int T, int H, int W);
cudaError_t launch_frame_scores(const void* x, int x_dtype, const void* y, int y_dtype, int B, int C, int T, int H, int W, float* psnr,
                                float* ssim, double* running, void* ws, cudaStream_t s);
// hi|lo split rows [rows][hi(C) | lo(C)] <-> fp32 rows [rows][C]
cudaError_t launch_split_to_f32(const bf16* x, float* y, long long rows, int C, cudaStream_t s);
cudaError_t launch_f32_to_split(const float* x, bf16* y, long long rows, int C, cudaStream_t s);

// conv_tc.cu (wgmma / TMA implicit GEMM)
// LayerNorm(+SiLU) of the output row fused into the conv epilogue (the row is complete in one N tile when Cout <= 256):
// mode 1: out := act(LN(v));  mode 2: out := v, out2 := act(LN(v))   (out2 uses the strides of out)
struct TcLnFusion {
  int mode = 0;
  bool silu = true;
  const float* gamma = nullptr;
  const float* beta = nullptr;
  void* out2 = nullptr;
};
// Regularizer fused into the epilogue of the encoder's conv_out (fp32 heads, Cout <= 32: the thread that owns an output
// position holds all of its channels): KL reparameterisation (distributions.py:8-18) or FSQ bound/round/index
// (regularizers.py:153-178), written straight to the caller's z / indices tensors ([B,zc,T,H,W] / [B,T,H,W]).
struct TcRegFusion {
  int mode = 0;                  // 0 none, 1 KL, 2 FSQ
  int zc = 0;
  int sample = 1;                // KL: z = mean + std * noise (else the mode)
  const float* noise = nullptr;  // KL, [B,zc,T,H,W]
  float* z = nullptr;
  int* indices = nullptr;        // FSQ (may be null)
  double* kl_acc = nullptr;      // KL: sum over all elements of mean^2 + var - 1 - logvar (cleared by the caller)
  int fsq_levels[VT_MAX_FSQ] = {0};
};
// One conv_tc launch as conv_tc_plan decides it (the tile fields are those of conv_tc.cu's TcParams)
struct TcPlan {
  ConvP p;
  DType tout;
  int w_batches, BN, BW, BH, BT, halo, hP, a_stages, stages, kparts, res_mma, ident_s;
  int stage_out;                 // bf16 output tiles leave through shared-memory staging buffers and bulk tensor stores
  int o_lo;                      // split output: channel offset of the lo plane from the output pointer (0: Co); a conv
                                 // that writes a channel slice of a wider tensor sets it to that tensor's channel count
  uint32_t halo_bytes, misc_off;
  size_t smem;
  TcLnFusion ln;                 // the requested epilogues that are taken (mode 0 otherwise)
  TcRegFusion reg;
};
// The wgmma plan of p with output type tout from geometry alone: no driver or runtime call, so a workspace dry run plans
// what the launch runs.  ln / reg request fused epilogues; one that does not fit is left out (mode 0) with the reason in
// conv_tc_last_error().  False, with the reason there, when conv_tc cannot run p.
bool conv_tc_plan(const ConvP& p, DType tout, const TcLnFusion* ln, const TcRegFusion* reg, int w_batches, TcPlan* out);
// w_nk: [Co_pad][K = taps * Cin] bf16 weights, w_batch_stride apart when batched; out may be null when a regularizer
// epilogue consumes the result.  A driver without cuTensorMapEncodeTiled is a launch error.
cudaError_t launch_conv_tc(const TcPlan& pl, const bf16* x, const bf16* w_nk, void* out, cudaStream_t s, long long w_batch_stride = 0);
// Makes the current device's residual identity tiles (bf16 and split) that res_mma launches read, if they do not exist yet;
// synchronises s when it makes them.  A launch that needs them while its stream is capturing fails instead of making them.
cudaError_t conv_tc_prepare_identity(cudaStream_t s);
cudaError_t launch_kl_clear(double* scratch, cudaStream_t s);
cudaError_t launch_kl_finish(const double* scratch, int B, float* kl_loss, cudaStream_t s);
// decoder head through per-tap partial outputs (see elementwise.cu)
cudaError_t launch_tap_planes_gather(const bf16* P, const float* bias, float* out, int B, int Ti, int H, int W, int NP, int Co,
                                     int to_off, cudaStream_t s, int pt = 2);
cudaError_t launch_pack_w_tap_planes(const float* w, bf16* out, int Co, int Ci, int NP, cudaStream_t s);
// x [batch][rows][cols] -> y [batch][cols][rows] (bf16), rows and cols multiples of 32
cudaError_t launch_transpose_bf16(const bf16* x, bf16* y, int batch, int rows, int cols, cudaStream_t s, bool split = false);
const char* conv_tc_last_error();

// tblock_tc.cu: ResnetCausalBlock1D (k311 conv -> LayerNorm -> SiLU -> k311 conv + residual) for C = 128, v1.0 padding
bool tblock_tc_supported(int B, int T, int H, int W, int C);
// Causal caches of a streamed video, bf16 [B,2,H,W,128] each: n1 = the block's input frames t-2, t-1, h = its LN2(h) frames
// (conv2's input).  *_in null: the first chunk (zero padding in front); *_out receive the chunk's last two frames and must
// not alias the inputs.
struct TbCache {
  const bf16* n1_in = nullptr;
  const bf16* h_in = nullptr;
  bf16* n1_out = nullptr;
  bf16* h_out = nullptr;
};
cudaError_t launch_tblock_tc(const bf16* n1, const bf16* x, const bf16* w1, const float* bias1, const float* gamma2,
                             const float* beta2, const bf16* w2, const float* bias2, bf16* out, bf16* out2,
                             const float* gamma_out, const float* beta_out, bool out_silu, int B, int T, int H, int W,
                             cudaStream_t s, const TbCache* cache = nullptr);
const char* tblock_tc_last_error();

// attn_tc.cu: fused per-frame attention O = softmax(Q K^T / sqrt(C)) V on wgmma with an online softmax (no tokens x tokens
// buffer).  q, k, v, o channels-last [frames, H*W, C] in bf16 or hi|lo split rows; C % 64 == 0, C <= 512, any token count.
// ws: attn_tc_workspace bytes (V^T, the size of v).
bool attn_tc_supported(long long frames, long long tokens, int C, bool split);
size_t attn_tc_workspace(long long frames, long long tokens, int C, bool split);
cudaError_t launch_attn_tc(const bf16* q, const bf16* k, const bf16* v, bf16* o, int frames, int H, int W, int C, bool split,
                           void* ws, cudaStream_t s);
const char* attn_tc_last_error();

// conv_stem.cu (thread-built im2col A tile + wgmma for the Cin=3 stem)
bool conv_stem_supported(const ConvP& p);
cudaError_t launch_conv_stem(const ConvP& p, const float* x, const bf16* wpk, bf16* out, cudaStream_t s);
cudaError_t launch_stem_cache_update(const float* x, float* cache, int B, int Ci, int T, int t_rep, int H, int W, cudaStream_t s);
// LPIPS stem: conv1_1 (3 -> 64, 1x3x3, ReLU) of 2 G images, frames [n0, n0 + G) of x then of y ([Bc,3,Tc,H,W], VT_DTYPE_*),
// with the evaluation script's preprocessing and LPIPS's ScalingLayer applied while loading; out channels-last [2G,H,W,64]
// (split: [2G,H,W,hi 64 | lo 64]); wpk as for launch_conv_stem (Kpad = 128, 9 taps)
cudaError_t launch_lpips_stem(const void* x, int x_dtype, const void* y, int y_dtype, int Tc, long long n0, int G, int H, int W,
                              bool split, const bf16* wpk, const float* bias, float acc_scale, bf16* out, cudaStream_t s);

// lpips.cu: the pooling and the per-position head of LPIPS (vidtok/modules/lpips.py) on channels-last features
// 2x2 / stride-2 max-pool (floor) of [N,H,W,C] (split: [N,H,W,hi C | lo C], compared as hi + lo) -> [N,H/2,W/2,C]
cudaError_t launch_maxpool2x2(const bf16* x, bf16* y, long long N, int H, int W, int C, bool split, cudaStream_t s);
// positions of one head tile, and the tiles of an H x W feature map
constexpr int kLpipsHeadPos = 64;
inline long long lpips_head_tiles(int H, int W) { return ((long long)H * W + kLpipsHeadPos - 1) / kLpipsHeadPos; }
// f [2G,H,W,C]: images [0,G) against [G,2G); part[g * tiles + tile] = sum over the tile's positions of
// sum_c w[c] (f_x / (|f_x| + 1e-10) - f_y / (|f_y| + 1e-10))^2, in fp32
cudaError_t launch_lpips_head(const bf16* f, int G, int H, int W, int C, bool split, const float* w, float* part, cudaStream_t s);
// per image g < G: layer k's partials (tiles[k] each, part + off[k]) added in order in double, / (H_k W_k), the five layers
// added in order; lpips[g] (fp32), per_layer[g][5] (may be null); running (may be null) += (sum of lpips[0..G), G)
struct LpipsFinish {
  long long off[5], tiles[5];
  double area[5];
};
cudaError_t launch_lpips_finish(const float* part, const LpipsFinish& f, int G, float* lpips, float* per_layer, double* running,
                                cudaStream_t s);

// Max-pool of channels-last [N,T,H,W,C] (split: hi C | lo C, compared as hi + lo) with SAME front padding (zeros) ->
// [N,To,Ho,Wo,C]; C % 8 == 0 (lpips.cu)
struct MaxPool3d {
  int T, H, W, C, To, Ho, Wo;
  int kt, kh, kw, st, sh, sw, pt, ph, pw;
};
cudaError_t launch_maxpool3d(const bf16* x, bf16* y, long long N, const MaxPool3d& q, bool split, cudaStream_t s);

// i3d.cu: the FVD feature network's own kernels.  Frames are resized so that the short side is 224 and centre-cropped to
// 224 x 224; Mixed_5c has 1024 channels and the logits 400.
constexpr int kI3dSize = 224, kI3dFeatC = 1024, kI3dClasses = 400;
struct I3dCrop { int Hr, Wr, oh, ow; };
inline I3dCrop i3d_crop(int H, int W) {
  I3dCrop c;
  // short side 224, long side ceil(long * 224 / short) in integers
  if (H <= W) { c.Hr = kI3dSize; c.Wr = (int)(((long long)W * kI3dSize + H - 1) / H); }
  else { c.Wr = kI3dSize; c.Hr = (int)(((long long)H * kI3dSize + W - 1) / W); }
  c.oh = (c.Hr - kI3dSize) / 2;
  c.ow = (c.Wr - kI3dSize) / 2;
  return c;
}
// clips [n0, n0 + G) of x [Bc,3,T,H,W] (VT_DTYPE_*) -> fp32 [G,3,T,224,224]: clamp, (v+1)/2, bilinear resize, crop, (v-0.5)*2
cudaError_t launch_i3d_resize(const void* x, int x_dtype, long long n0, int G, int T, int H, int W, float* out, cudaStream_t s);
// Conv3d_1a_7x7 with folded BatchNorm and ReLU: x [G,3,T,224,224] fp32 -> channels-last [G,To,112,112,64] (split: hi|lo);
// wpk [64][1088] (launch_pack_w_nk_bf16, 343 taps, Kpad 1088) or its split copy
size_t i3d_stem_smem(bool split);
cudaError_t launch_i3d_stem(const float* x, int G, int T, int To, int pt, int ph, int pw, bool split, const bf16* wpk, const float* bias,
                            float acc_scale, bf16* out, cudaStream_t s);
// Mixed_5c [G,T5,7,7,1024] -> features [G,400]: AvgPool3d [2,7,7], the logits (wt [1024][400] fp32, bias [400]), mean over time
cudaError_t launch_i3d_head(const bf16* f, int G, int T5, bool split, const float* wt, const float* bias, float* feat, cudaStream_t s);
// stats [1 + 400 + 400 * 400] doubles += (G, sum f, sum f f^T), clip by clip in index order
cudaError_t launch_i3d_stats(const float* feat, int G, double* stats, cudaStream_t s);
// Real channel c of a stored layout: in segment k (real0 <= c < real0 + count) it is stored at stored0 + c - real0
struct I3dSegs {
  int n, real;
  int real0[4], stored0[4], count[4];
};
cudaError_t launch_i3d_unpack(const bf16* x, bool split, long long N, int T, int H, int W, int Cs, const I3dSegs& segs, float* out,
                              cudaStream_t s);

}  // namespace vt
