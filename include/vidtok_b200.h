/*
 * vidtok_b200 -- C ABI of the H100-native (sm_90a) VidTok causal tokenizer hot path
 * (encode -> KL/FSQ regularize -> decode).
 *
 * The reference (microsoft/VidTok @ d6ad92d) has no FFI / plugin registry: the only indirection on this
 * path is `instantiate_from_config` (vidtok/modules/util.py:69-86), which builds
 * vidtok.models.autoencoder[_v1_1].AutoencodingEngine from a YAML `target:` string, and the engine's
 * encode()/decode()/forward() methods (vidtok/models/autoencoder.py:197-229,
 * vidtok/models/autoencoder_v1_1.py:230-342).  The entry points below are what a binding for THAT
 * interface needs: one opaque model handle per (config, device), a parameter manifest that uses the
 * reference's checkpoint key names, and encode/decode calls that take raw device pointers in the
 * reference's tensor layout ([B,C,T,H,W], fp32).  INTEGRATION.md shows the ctypes binding.
 *
 * Conventions: plain C types only; every function returns 0 on success or a negative vt_status and
 * records a message retrievable with vt_last_error() (thread-local).  The library never allocates
 * caller-visible outputs: the caller owns inputs, outputs and the scratch workspace (size queried
 * first).  All device work is enqueued on the caller's cudaStream_t (passed as void*); calls on one
 * handle must be serialised by the caller (the reference's modules are not re-entrant either:
 * chunk caches live on the modules, vidtok/modules/model_3dcausal_v1_1.py:155-157).
 */
#ifndef VIDTOK_B200_H
#define VIDTOK_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VT_MAX_LEVELS 8

typedef enum {
  VT_OK = 0,
  VT_ERR_INVALID = -1,    /* bad argument / unsupported configuration */
  VT_ERR_CUDA = -2,       /* CUDA runtime or driver error */
  VT_ERR_NOT_READY = -3,  /* parameters missing or vt_model_finalize not called */
  VT_ERR_WORKSPACE = -4,  /* workspace too small */
  VT_ERR_NO_DEVICE = -5,  /* no sm_90a (H100) device: there is deliberately no CPU fallback */
  VT_ERR_CAPTURE = -6     /* the caller's stream is capturing a CUDA graph and the call would allocate, synchronise or
                             copy from host memory (see "CUDA graph capture" below); nothing was enqueued */
} vt_status;

/* Precision modes.
 * EXACT_TC (the parity mode): fp32-class results on the tensor cores (wgmma).  Activations and weights are kept as
 *   two fp16 planes (hi = fp16(v), lo = fp16(v - hi): 11 + 11 mantissa bits); every K step issues hi*hi + lo*hi + hi*lo
 *   into the fp32 register accumulator ("fp16x3": products good to ~2^-21), LayerNorm / SiLU / regularizers in fp32.
 *   Gate: 1e-3 max-abs, FSQ codes equal.
 * BF16 (the throughput mode): bf16 activations / weights, fp32 accumulation.  Gate: PSNR within 0.01 dB.
 * MIXED: encoder in EXACT_TC (bit-exact FSQ codes / 1e-3 latents), decoder in BF16.
 * FMA32 (VT_PREC_EXACT, kept for cross-checks): fp32 activations on fp32 FMA kernels, no tensor cores. */
#define VT_PREC_EXACT 0
#define VT_PREC_FMA32 0
#define VT_PREC_BF16 1
#define VT_PREC_EXACT_TC 2
#define VT_PREC_MIXED 3

#define VT_NORM_LAYERNORM 0
#define VT_NORM_GROUPNORM 1
#define VT_REG_KL 0
#define VT_REG_FSQ 1
#define VT_INTERP_NEAREST 0
#define VT_INTERP_TRILINEAR 1

/* Mirrors the `encoder_config.params` block of configs/STAR.yaml plus the regularizer choice
 * (e.g. configs/vidtok_kl_causal_488_4chn.yaml:11-36).  n_* == -1 selects the reference default
 * (vidtok/modules/model_3dcausal.py:539-540,756-757). */
typedef struct vt_model_desc {
  int32_t version;                /* 0 = v1.0 (model_3dcausal.py), 1 = v1.1 (model_3dcausal_v1_1.py) */
  int32_t ch;
  int32_t num_levels;             /* len(ch_mult) */
  int32_t ch_mult[VT_MAX_LEVELS];
  int32_t num_res_blocks;
  int32_t in_channels;
  int32_t out_ch;
  int32_t z_channels;
  int32_t double_z;
  int32_t norm_type;              /* VT_NORM_* */
  int32_t time_downsample_factor;
  int32_t n_spatial_ds, spatial_ds[VT_MAX_LEVELS];
  int32_t n_tempo_ds, tempo_ds[VT_MAX_LEVELS];
  int32_t n_spatial_us, spatial_us[VT_MAX_LEVELS];
  int32_t n_tempo_us, tempo_us[VT_MAX_LEVELS];
  int32_t interpolation_mode;     /* VT_INTERP_* (v1.1 only) */
  int32_t regularizer;            /* VT_REG_* */
  int32_t fsq_num_levels;
  int32_t fsq_levels[VT_MAX_LEVELS];
  int32_t kl_sample;              /* DiagonalGaussianRegularizer(sample=...) regularizers.py:75 */
  int32_t noncausal;              /* 1 = the non-causal family (vidtok/modules/model_3dnoncausal.py: Encoder3D / Decoder3D; v1.0
                                     only): symmetric zero padding in time, plain nn.Conv3d/1d checkpoint keys, no front
                                     padding of the clip, no dropped frames */
} vt_model_desc;

typedef struct vt_model vt_model;

const char* vt_last_error(void);
int32_t vt_abi_version(void);
/* number of kernels launched by this library on this thread since the last call with reset != 0 */
int64_t vt_launch_count(int32_t reset);

/* Optional per-kernel profile of everything this thread launches between start and stop: CUDA events on the launch
 * stream around every kernel (adds launch gaps: use it to attribute time, not to measure throughput).
 * vt_profile_stop waits for the profiled kernels (their events, not the device) and writes a JSON object
 * {"kernel": {"launches": n, "ms": total, "flops": algorithmic, "bytes": algorithmic}, ...}; returns its length. */
void vt_profile_start(void);
void vt_profile_start_detailed(void); /* keys additionally carry the layer geometry */
int32_t vt_profile_stop(char* json, int32_t cap);

/* ---- model lifetime (replaces AutoencodingEngine.__init__, autoencoder.py:103-144) ---- */
int32_t vt_model_create(const vt_model_desc* desc, int32_t device, vt_model** out);
void vt_model_destroy(vt_model* m);

/* Parameter manifest: names are the reference checkpoint keys ("encoder.conv_in.conv.weight", ...;
 * SURVEY.md section 8b), shapes are the reference's (OIDHW / OIHW / OIW / [C] / [1]). */
int32_t vt_model_num_params(const vt_model* m);
int32_t vt_model_param_info(const vt_model* m, int32_t index, char* name, int32_t name_cap, int64_t* shape5,
                            int32_t* ndim);
/* Copies one fp32 parameter (host or device pointer, `numel` floats) into the model
 * (replaces load_state_dict, autoencoder.py:164). */
int32_t vt_model_load_param(vt_model* m, const char* name, const float* data, int64_t numel, int32_t is_device,
                            void* stream);
/* Repacks all parameters for the kernels (K-major bf16 tiles for wgmma, [K][Cout] fp32 for the FMA
 * path).  Must be called after the last vt_model_load_param and before encode/decode. */
int32_t vt_model_finalize(vt_model* m, void* stream);

/* ---- whole-clip path (AutoencodingEngine.encode/decode, autoencoder.py:197-219;
 *      untiled v1.1: autoencoder_v1_1.py:230-241,286-300) ---- */
/* Latent geometry for an input of T x H x W: frames (after the encoder's front padding), height, width. */
int32_t vt_latent_shape(const vt_model* m, int32_t T, int32_t H, int32_t W, int32_t* Tz, int32_t* Hz, int32_t* Wz);
/* Number of frames decode() returns for Tz latent frames (v1.0 drops tdf-1, model_3dcausal.py:885). */
int32_t vt_decoded_frames(const vt_model* m, int32_t Tz);
int64_t vt_workspace_bytes(const vt_model* m, int32_t precision, int32_t B, int32_t T, int32_t H, int32_t W);

/* x: device fp32 [B,C,T,H,W]; C must equal in_channels (a mismatch is rejected: the reference raises a shape error in
 * conv_in, model_3dcausal.py:634).  noise: device fp32 [B,z,Tz,Hz,Wz] = the reference's
 * torch.randn(mean.shape) (distributions.py:17), required for KL with kl_sample, else NULL.
 * Outputs (device, caller-allocated): z fp32 [B,z,Tz,Hz,Wz]; indices int32 [B,Tz,Hz,Wz] (FSQ, may be
 * NULL); kl_loss 1 float (KL, may be NULL); h_pre fp32 [B,2z|z,Tz,Hz,Wz] encoder output before the
 * regularizer (may be NULL). */
int32_t vt_encode(vt_model* m, int32_t precision, const float* x, int32_t B, int32_t C, int32_t T, int32_t H, int32_t W,
                  const float* noise, float* z, int32_t* indices, float* kl_loss, float* h_pre, void* workspace,
                  int64_t workspace_bytes, void* stream);
/* z: device fp32 [B,Cz,Tz,Hz,Wz] with Cz == z_channels, or (from_indices; Cz ignored) int32 [B,Tz,Hz,Wz]
 * (autoencoder.py:205-217).
 * x_out: device fp32 [B,out_ch,vt_decoded_frames(Tz),Hz*s,Wz*s]. */
int32_t vt_decode(vt_model* m, int32_t precision, const void* z, int32_t from_indices, int32_t B, int32_t Cz, int32_t Tz,
                  int32_t Hz, int32_t Wz, float* x_out, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- temporal tiling with causal caches (v1.1: tile_encode / tile_decode,
 *      autoencoder_v1_1.py:244-264,302-331; per-layer caches model_3dcausal_v1_1.py:159-178,216-236,
 *      289-302,325-343).  One state object per in-flight video.
 *      Causal v1.0 models stream through the same calls: the first chunk has 1 (mod tdf) frames (it gets the tdf-1
 *      replicated front frames and zero time padding, model_3dcausal.py:680-688), later chunks whole multiples of tdf;
 *      decoding drops tdf-1 frames of the first chunk only (:883-885).  Every v1.0 norm and attention works within one
 *      frame, so the concatenated chunk outputs equal the whole-clip encode / decode (bit for bit in VT_PREC_BF16 and
 *      VT_PREC_FMA32; to fp32 rounding in the split-operand mode).  use_overlap is v1.1
 *      only; non-causal models are rejected (a frame depends on later frames).  A v1.0 decoder state takes latents. ---- */
typedef struct vt_chunk_state vt_chunk_state;
int32_t vt_chunk_state_create(vt_model* m, int32_t precision, int32_t B, int32_t H, int32_t W, int32_t is_decoder,
                              int32_t use_overlap, vt_chunk_state** out);
void vt_chunk_state_destroy(vt_chunk_state* s);
int64_t vt_chunk_workspace_bytes(const vt_chunk_state* s, int32_t T_chunk);
/* x_chunk: device fp32 [B,C,Tc,H,W] (dense), C == in_channels.  Outputs as vt_encode, for this chunk only. */
int32_t vt_encode_chunk(vt_chunk_state* s, int32_t is_first, const float* x_chunk, int32_t C, int32_t Tc, const float* noise,
                        float* z, int32_t* indices, float* kl_loss, void* workspace, int64_t workspace_bytes,
                        void* stream);
/* vt_encode_chunk that also writes the chunk's encoder output before the regularizer, h_pre device fp32 [B,2z|z,Tz,Hz,Wz]
 * (per-sample losses of a batched state: each sample's KL loss or FSQ aux partials); z / indices as vt_encode_chunk. */
int32_t vt_encode_chunk_pre(vt_chunk_state* s, int32_t is_first, const float* x_chunk, int32_t C, int32_t Tc, const float* noise,
                            float* z, int32_t* indices, float* kl_loss, float* h_pre, void* workspace, int64_t workspace_bytes,
                            void* stream);
/* vt_encode_chunk of an FSQ model that also writes this chunk's partials of the FSQ aux loss (see vt_fsq_aux_partials):
 * stats fp32 [2] and avg_prob fp32 [J], J = prod(levels), over the chunk's B * Tz * Hz * Wz tokens -- the per-chunk step of
 * vt_encode_video_fsq_aux.  The workspace holds the chunk's pre-bound latent and the partials' scratch on top of
 * vt_chunk_workspace_bytes; vt_chunk_fsq_aux_workspace_bytes returns -1 (and records why) for a decoder state, a KL model or
 * a level list vt_fsq_aux_partials does not support, and vt_encode_chunk_fsq_aux fails with VT_ERR_INVALID before any launch. */
int64_t vt_chunk_fsq_aux_workspace_bytes(const vt_chunk_state* s, int32_t T_chunk);
int32_t vt_encode_chunk_fsq_aux(vt_chunk_state* s, int32_t is_first, const float* x_chunk, int32_t C, int32_t Tc, float* z,
                                int32_t* indices, float inv_temperature, float* stats, float* avg_prob, void* workspace,
                                int64_t workspace_bytes, void* stream);
/* z_chunk: device fp32 [B,Cz,Tzc,Hz,Wz] (Cz == z_channels) including the look-ahead frame when overlap applies; x_out receives
 * all decoded frames of this chunk (the caller trims the look-ahead tail as autoencoder_v1_1.py:327-328). */
int32_t vt_decode_chunk(vt_chunk_state* s, int32_t is_first, const float* z_chunk, int32_t Cz, int32_t Tzc, float* x_out,
                        void* workspace, int64_t workspace_bytes, void* stream);
/* Slot transplant: for every cache src holds, copies the readable cache of batch slot src_slots[i] of src into slot
 * dst_slots[i] of dst (host arrays of n slots), in one launch on `stream`.  The caches are the whole state a chunk carries
 * to the next (is_first is an argument of each chunk call, the overlap decoder's cache offsets depend on the cache key
 * alone), so after the copy dst slot dst_slots[i] is the state the src slot would have had: the next non-first chunk
 * computes in that slot what it would have computed in src's.  Caches dst does not hold yet are allocated for dst's batch
 * (zeroed) and every cache filled is marked written.  Refused with VT_ERR_INVALID, before anything is enqueued: states of
 * different models, precisions, H x W, direction or use_overlap, the same state as both ends, slots out of range, a dst
 * slot listed twice, or a cache whose per-slot size differs between the two.  Calls on one dst state must use one stream. */
int32_t vt_chunk_state_copy_slots(vt_chunk_state* dst, const vt_chunk_state* src, int32_t n, const int32_t* dst_slots,
                                  const int32_t* src_slots, void* stream);

/* ---- CUDA graph capture.  vt_encode, vt_decode, vt_encode_chunk, vt_encode_chunk_pre, vt_encode_chunk_fsq_aux and
 *      vt_decode_chunk may be captured into a CUDA graph on the caller's stream: they launch kernels and stream-ordered
 *      memsets only, with every tensor map and launch parameter fixed at capture.  State a call may create must exist before
 *      capture: the residual identity tiles (made by vt_model_finalize) and, for a chunk state, both buffers of every cache a
 *      chunk of that length uses (vt_chunk_state_reserve).  Each entry point asks cudaStreamIsCapturing of `stream`; when
 *      it is capturing and the call would allocate, synchronise or copy from host memory, it returns VT_ERR_CAPTURE before
 *      anything is enqueued and vt_last_error() names what was missing.  Refused under capture: vt_encode_video,
 *      vt_decode_video and vt_encode_video_fsq_aux (library copy stream, host staging), vt_chunk_state_copy_slots (uploads
 *      a host table), any call while the profiler is on, and a chunk whose caches were not reserved.
 *      A captured chunk is only valid for the cache parity it was captured at: it reads buffer `parity` and writes the other
 *      one of every cache.  Capturing updates the state as running the chunk would (its caches flip); a replay of that graph
 *      must be followed by vt_chunk_state_advance, with no other chunk call on the state in between. ---- */
/* Allocates (or takes from the model's pool) and zeroes both buffers of every cache a chunk of T_chunk frames (encoder) or
 * latent frames (decoder) uses, found by the dry run of vt_chunk_workspace_bytes; caches already held at that size are left
 * as they are.  The zeroing is enqueued on `stream`, which must not be capturing (VT_ERR_CAPTURE).  After it, chunks of that
 * length run under capture. */
int32_t vt_chunk_state_reserve(vt_chunk_state* s, int32_t T_chunk, void* stream);
/* The cur bit of the state's double-buffered caches (every cache commits on every chunk, so they agree): 0 or 1, 0 for a
 * state that holds no cache yet, -1 (and a message) for a null state or caches that disagree. */
int32_t vt_chunk_state_parity(const vt_chunk_state* s);
/* Marks one chunk as run outside the library, by the replay of a graph captured at the current parity: every cache flips
 * its parity and counts as written, as the chunk call itself would have left them.  Enqueues nothing. */
int32_t vt_chunk_state_advance(vt_chunk_state* s);

/* ---- whole-video tiling below the ABI (tile_encode / tile_decode, autoencoder_v1_1.py:218-228,244-264,302-331): the chunk
 *      schedule, the causal caches and the chunk staging run inside the library -- one call per video, no host
 *      synchronisation, no per-chunk allocation.  Chunk i+1 is staged on the library's own copy stream while chunk i
 *      computes on the caller's stream (double buffering); with x_on_host / out_on_host the staging copies are the
 *      host <-> device transfers themselves (pinned memory recommended).  The call returns with all work enqueued; the
 *      caller's stream is made to wait for the copy stream. ---- */
int64_t vt_encode_video_workspace_bytes(const vt_model* m, int32_t precision, int32_t B, int32_t T, int32_t H, int32_t W,
                                        int32_t t_chunk_enc);
/* x fp32 [B,C,T,H,W] (device, or host when x_on_host); noise device fp32 [B,z,Tz,Hz,Wz] = the per-chunk torch.randn draws
 * concatenated along T (KL with sampling; else NULL); z / indices as vt_encode for the whole video (Tz = sum of the chunks'
 * latent frames); kl_loss = mean of the per-chunk values (autoencoder_v1_1.py:261-264). */
int32_t vt_encode_video(vt_model* m, int32_t precision, const float* x, int32_t x_on_host, int32_t B, int32_t C, int32_t T,
                        int32_t H, int32_t W, int32_t t_chunk_enc, const float* noise, float* z, int32_t* indices,
                        float* kl_loss, void* workspace, int64_t workspace_bytes, void* stream);
/* vt_encode_video of an FSQ model that also writes the per-chunk partials of the FSQ aux loss (see vt_fsq_aux_partials):
 * chunk i of the schedule (first frame alone, then t_chunk_enc frames each) writes aux_stats[2i..2i+1] and
 * aux_avg_prob[i*J .. (i+1)*J), J = prod(levels).  z / indices as vt_encode_video; host-staged and device inputs give the
 * same bits.  The workspace is larger than vt_encode_video's. */
int64_t vt_encode_video_fsq_aux_workspace_bytes(const vt_model* m, int32_t precision, int32_t B, int32_t T, int32_t H, int32_t W,
                                                int32_t t_chunk_enc);
int32_t vt_encode_video_fsq_aux(vt_model* m, int32_t precision, const float* x, int32_t x_on_host, int32_t B, int32_t C, int32_t T,
                                int32_t H, int32_t W, int32_t t_chunk_enc, float* z, int32_t* indices, float inv_temperature,
                                float* aux_stats, float* aux_avg_prob, void* workspace, int64_t workspace_bytes, void* stream);
int64_t vt_decode_video_workspace_bytes(const vt_model* m, int32_t precision, int32_t B, int32_t Tz, int32_t Hz, int32_t Wz,
                                        int32_t t_chunk_dec, int32_t use_overlap);
/* frames vt_decode_video writes (look-ahead tails dropped; the v1.1 forward then keeps the last T_in frames) */
int32_t vt_decode_video_frames(const vt_model* m, int32_t Tz, int32_t t_chunk_dec, int32_t use_overlap);
/* z device fp32 [B,Cz,Tz,Hz,Wz]; x_out fp32 [B,out_ch,vt_decode_video_frames(...),H,W] (device, or host when out_on_host) */
int32_t vt_decode_video(vt_model* m, int32_t precision, const float* z, int32_t B, int32_t Cz, int32_t Tz, int32_t Hz, int32_t Wz,
                        int32_t t_chunk_dec, int32_t use_overlap, float* x_out, int32_t out_on_host, void* workspace,
                        int64_t workspace_bytes, void* stream);

/* Temporal reach R of a causal v1.1 model under the tile_encode / tile_decode chunking: an output frame depends on no input
 * more than R frames before it.  Encoder (is_decoder 0): latent l depends on input frames >= f - R, f = its group's first
 * frame (0 for l = 0, else 1 + (l-1) * tdf).  Decoder: decoded frame t depends on latent frames >= t / tdf - R; use_overlap
 * selects the look-ahead chunking (its caches hold the frames before each chunk; without overlap the trilinear time
 * upsample's cache reaches further back).  Composed from the layer list the executor runs; no device is touched.
 * VT_ERR_INVALID for v1.0 and non-causal models, and for use_overlap on the encoder. */
int32_t vt_temporal_reach(const vt_model* m, int32_t is_decoder, int32_t use_overlap, int32_t* frames);

/* ---- video I/O adjacent steps (scripts/inference_reconstruct.py:41-47,71-82,231-239): the tokenizer runs at > 1000
 *      frames/s, so the uint8 <-> float conversions around it belong on the device too ---- */
/* frames: device uint8 [T,Hs,Ws,C] (decord's HWC frames); clip: device fp32 [C,T,H,W] = Normalize(.5,.5)(frames/255)
 * of the crop window at (h0, w0) (CenterCrop; the optional Resize is not part of this entry point). */
int32_t vt_video_u8_to_clip(const uint8_t* frames, float* clip, int32_t T, int32_t Hs, int32_t Ws, int32_t C, int32_t h0,
                            int32_t w0, int32_t H, int32_t W, void* stream);
/* frames: device uint8 [N,Hs,Ws,C]; clip: device fp32 [N/Tc,C,Tc,H,W], frame n -> clip n/Tc, time n%Tc.  The reference's
 * Resize(antialias=True) -> CenterCrop -> Normalize(.5,.5) of frames/255: torch's antialiased bilinear resize to Hr x Wr
 * (align_corners=False), then the crop window at (h0, w0), in one launch without workspace.  N % Tc == 0 and the window
 * must lie inside Hr x Wr.  VT_ERR_INVALID when the downscale is so large that the source window of one output pixel
 * does not fit in shared memory (about 130x for C = 3). */
int32_t vt_video_u8_to_clip_resized(const uint8_t* frames, float* clip, int32_t N, int32_t Hs, int32_t Ws, int32_t C, int32_t Hr,
                                    int32_t Wr, int32_t h0, int32_t w0, int32_t H, int32_t W, int32_t Tc, void* stream);
/* clip: device fp32 [C,T,H,W]; frames: device uint8 [T,H,W,C] = uint8(255 * (clamp(clip,-1,1) + 1) / 2) (tensor_to_uint8). */
int32_t vt_clip_to_video_u8(const float* clip, uint8_t* frames, int32_t C, int32_t T, int32_t H, int32_t W, void* stream);

/* ---- scoring a reconstruction (scripts/inference_evaluate.py:175-186 with compute_psnr / compute_ssim,
 *      vidtok/modules/util.py:146-231): clamp to [-1,1], (v+1)/2, then per frame PSNR = -10 log10(mean squared error over
 *      C x H x W + 1e-8) and SSIM = mean over channels of the mean SSIM map (frames average-pooled by
 *      max(1, round(min(H,W)/256)) first, round half to even; 11 x 11 Gaussian window, sigma 1.5, no padding; c1 = 1e-4,
 *      c2 = 9e-4), in one pass over the two clips.  The mean of the per-frame values over a video equals the script's mean
 *      over its groups of 16 frames, each group value repeated once per frame.  The script clamps only the reconstruction;
 *      here x is clamped as well, which changes nothing for an input clip in [-1,1].  Every sum runs in a fixed order:
 *      repeated calls give the same bits. ---- */
#define VT_DTYPE_F32 0
#define VT_DTYPE_BF16 1
#define VT_DTYPE_F16 2
/* bytes of workspace for one call at this geometry; -1 (and a message) for an empty shape or more tiles than one launch holds */
int64_t vt_frame_scores_workspace_bytes(int32_t B, int32_t C, int32_t T, int32_t H, int32_t W);
/* x (the input clip) and y (the reconstruction, not yet clamped): device, dense [B,C,T,H,W], each VT_DTYPE_*; a batch of
 * frames [N,C,H,W] is B = N, T = 1.  psnr, ssim: device fp32 [B*T], frame (b, t) at b*T + t.  ssim may be NULL (PSNR only);
 * otherwise the pooled frame must be at least 11 x 11 (VT_ERR_INVALID, as the reference raises ValueError).  running (device,
 * may be NULL): three doubles that receive += (sum of this call's PSNR values, sum of its SSIM values when ssim is given,
 * B*T), added frame by frame in order, so a video scored in several calls on one stream needs no host synchronisation
 * and accumulates the same bits as one call. */
int32_t vt_frame_scores(const void* x, int32_t x_dtype, const void* y, int32_t y_dtype, int32_t B, int32_t C, int32_t T, int32_t H,
                        int32_t W, float* psnr, float* ssim, double* running, void* workspace, int64_t workspace_bytes,
                        void* stream);

/* ---- LPIPS of a reconstruction (vidtok/modules/lpips.py, scripts/inference_evaluate.py:175-186): per frame, the script's
 *      clamp of the reconstruction, (v+1)/2 then *2-1, LPIPS's ScalingLayer, VGG16 features[0:30] (13 3x3 ReLU convolutions
 *      and four 2x2 max-pools) and the head of the five taps relu1_2 .. relu5_3 (channel-normalised squared difference,
 *      lin_k, mean over the tap's H x W, the five layers added).  One handle holds the weights, built like vt_model.  The
 *      frame pairs run in passes of vt_lpips_pass_frames(H, W) pairs; a frame's value does not depend on the pass or the
 *      call it falls into, and every sum runs in a fixed order: repeated calls give the same bits. ---- */
typedef struct vt_lpips_model vt_lpips_model;
int32_t vt_lpips_create(int32_t device, vt_lpips_model** out);
void vt_lpips_destroy(vt_lpips_model* h);
/* The reference's state-dict keys and shapes: net.slice{1..5}.{i}.weight [Co,Ci,3,3] / .bias [Co] for i in 0, 2 | 5, 7 |
 * 10, 12, 14 | 17, 19, 21 | 24, 26, 28, and lin{0..4}.model.1.weight [1,C,1,1].  The ScalingLayer's constant buffers are not
 * parameters. */
int32_t vt_lpips_num_params(const vt_lpips_model* h);
int32_t vt_lpips_param_info(const vt_lpips_model* h, int32_t index, char* name, int32_t name_cap, int64_t* shape4, int32_t* ndim);
int32_t vt_lpips_load_param(vt_lpips_model* h, const char* name, const float* data, int64_t numel, int32_t is_device, void* stream);
/* repacks the convolutions for the kernels (bf16, and the split copy of EXACT_TC); after the last load, before vt_lpips_model */
int32_t vt_lpips_finalize(vt_lpips_model* h, void* stream);
/* frame pairs per pass at H x W: 16, or fewer where relu1_2 of a pass (2 images per pair x H x W x 64) would exceed 2^31
 * elements; 0 when not even one pair fits */
int32_t vt_lpips_pass_frames(int32_t H, int32_t W);
/* workspace of vt_lpips for this geometry (one pass: two activation buffers and the heads' partials); -1 and a message for a
 * geometry vt_lpips refuses */
int64_t vt_lpips_workspace_bytes(const vt_lpips_model* h, int32_t precision, int32_t B, int32_t C, int32_t T, int32_t H, int32_t W);
/* x (the input clip) and y (the reconstruction, not yet clamped): device, dense [B,C,T,H,W], each VT_DTYPE_*; frames [N,C,H,W]
 * are B = N, T = 1.  precision: VT_PREC_BF16 or VT_PREC_EXACT_TC.  C must be 3 and H, W at least 16 (relu5_3 at least 1 x 1);
 * otherwise VT_ERR_INVALID and nothing is launched.  lpips: device fp32 [B*T]; per_layer (device, may be NULL): fp32
 * [B*T][5], the five layers' terms; running (device, may be NULL): two doubles that receive += (sum of this call's values,
 * B*T), frame by frame in order. */
int32_t vt_lpips(vt_lpips_model* h, int32_t precision, const void* x, int32_t x_dtype, const void* y, int32_t y_dtype, int32_t B, int32_t C,
                 int32_t T, int32_t H, int32_t W, float* lpips, float* per_layer, double* running, void* workspace,
                 int64_t workspace_bytes, void* stream);

/* ---- I3D features for the Frechet video distance (FVD).  The definition (vidtok_b200/metrics.py, README "FVD"): each clip
 *      clamped to [-1,1], (v+1)/2, every frame resized bilinearly (align_corners=False, no antialias) to short side 224 and
 *      long side ceil(long * 224 / short), centre-cropped to 224 x 224, (v-0.5)*2; I3D (Inception-v1 inflated, Kinetics-400,
 *      the PyTorch port's InceptionI3d layout); the 400 logits averaged over the remaining time steps.  One handle holds the
 *      weights, built like vt_lpips_model.  Clips run in passes of vt_i3d_pass_clips(T, H, W); a clip's features do not depend
 *      on the pass or the call, and every sum runs in a fixed order. ---- */
typedef struct vt_i3d_model vt_i3d_model;
int32_t vt_i3d_create(int32_t device, vt_i3d_model** out);
void vt_i3d_destroy(vt_i3d_model* h);
/* The port's state-dict keys: <unit>.conv3d.weight [Co,Ci,k,k,k] and <unit>.bn.{weight,bias,running_mean,running_var} [Co]
 * for Conv3d_1a_7x7, Conv3d_2b_1x1, Conv3d_2c_3x3 and Mixed_{3b,3c,4b,4c,4d,4e,4f,5b,5c}.{b0,b1a,b1b,b2a,b2b,b3b};
 * logits.conv3d.weight [400,1024,1,1,1] and logits.conv3d.bias [400].  shape5: five extents (1 beyond ndim). */
int32_t vt_i3d_num_params(const vt_i3d_model* h);
int32_t vt_i3d_param_info(const vt_i3d_model* h, int32_t index, char* name, int32_t name_cap, int64_t* shape5, int32_t* ndim);
int32_t vt_i3d_load_param(vt_i3d_model* h, const char* name, const float* data, int64_t numel, int32_t is_device, void* stream);
/* folds BatchNorm (eps 1e-3) into the weights, packs them for the kernels (bf16 and the split copy of EXACT_TC); synchronises */
int32_t vt_i3d_finalize(vt_i3d_model* h, void* stream);
/* clips per pass for T frames: 8, or fewer where an activation of the pass would exceed 2^31 elements; 0 for T < 9 */
int32_t vt_i3d_pass_clips(const vt_i3d_model* h, int32_t T, int32_t H, int32_t W);
/* workspace of vt_i3d_features for this geometry (one pass); -1 and a message for a geometry it refuses */
int64_t vt_i3d_workspace_bytes(const vt_i3d_model* h, int32_t precision, int32_t B, int32_t C, int32_t T, int32_t H, int32_t W);
/* x: device, dense [B,C,T,H,W] of VT_DTYPE_*, in [-1,1].  precision VT_PREC_BF16 or VT_PREC_EXACT_TC; C must be 3 and T at
 * least 9, otherwise VT_ERR_INVALID and nothing is launched.  features: device fp32 [B,400].  stats (device, may be NULL):
 * doubles [n, sum f (400), sum f f^T (400 x 400)] that receive += this call's clips, clip by clip in index order. */
int32_t vt_i3d_features(vt_i3d_model* h, int32_t precision, const void* x, int32_t x_dtype, int32_t B, int32_t C, int32_t T, int32_t H,
                        int32_t W, float* features, double* stats, void* workspace, int64_t workspace_bytes, void* stream);
/* For the tests: the activation at end point `name` (Conv3d_1a_7x7 ... Mixed_5c, the port's names) of up to one pass of
 * clips, as fp32 [B,C,T,H,W] of the real channels into out.  shape5 (may be NULL) receives that shape; with out NULL only the
 * shape is computed and nothing is launched. */
int32_t vt_i3d_endpoint(vt_i3d_model* h, int32_t precision, const void* x, int32_t x_dtype, int32_t B, int32_t C, int32_t T, int32_t H,
                        int32_t W, const char* name, float* out, int64_t* shape5, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- single operators, exposed for the parity tests (same kernels the model path launches) ---- */
typedef struct vt_conv_desc {
  int32_t B, Ti, Hi, Wi, Ci;        /* input, channels-last [B,Ti,Hi,Wi,Ci] */
  int32_t Co, kt, kh, kw;
  int32_t st, sh, sw;               /* strides */
  int32_t pt;                       /* causal front pad in time (zeros) */
  int32_t ph0, ph1, pw0, pw1;       /* spatial zero pads (top,bottom,left,right) */
  int32_t ut, uh, uw;               /* nearest-neighbour upsampling of the input folded into the gather */
  int32_t res_mode;                 /* 0 none, 1 out = conv + res, 2 out = a*res[t/2] + (1-a)*conv, 3 out = a*avgpool3(res) + (1-a)*conv */
  float alpha;
} vt_conv_desc;
/* x/res/out are channels-last activations in the precision's activation type: fp32 (FMA32), bf16 (BF16), or hi|lo split
 * bf16 rows [..., hi(C) | lo(C)] (EXACT_TC; value = hi + lo); w fp32 [Co,Ci,kt,kh,kw]; bias fp32 [Co].
 * BF16 / EXACT_TC run the wgmma kernel (an unsupported geometry is an error, never a silent fallback) unless
 * force_simt != 0, which runs the fp32-FMA kernel on the same operands. */
int32_t vt_op_conv(int32_t precision, int32_t force_simt, const vt_conv_desc* d, const void* x, const float* w,
                   const float* bias, const void* res, void* out, void* stream);
/* The variants of the convolution the model path uses beyond vt_conv_desc: v1.1 time padding (replicated first frame /
 * per-layer cache, model_3dcausal_v1_1.py:216-236), LayerNorm(+SiLU) fused into the epilogue (model_3dcausal.py:62-80),
 * dropped leading output frames (:883-885), fp32 [B,C,T,H,W] output (the heads), residual as a mix. */
typedef struct vt_conv_ex {
  vt_conv_desc d;
  int32_t force_simt;
  int32_t t_mode;          /* 0 zeros, 1 replicate frame 0, 2 `cache` holds cacheT frames [B,cacheT,H,W,C] in front of x */
  int32_t cacheT;
  int32_t ln_mode;         /* 0 none, 1 out := act(LN(v)), 2 out := v and out2 := act(LN(v)) */
  int32_t ln_silu;
  int32_t to_off;          /* leading output frames dropped */
  int32_t out_f32_ncdhw;   /* out is fp32 [B,Co,To,Ho,Wo] */
  int32_t res_mix;         /* res_mode 1 computes alpha*res + (1-alpha)*conv instead of res + conv */
  int32_t res_t_mode;      /* res_mode 3 front pad: 0 zero, 1 frame 0, 2 `cache` = 1 frame [B,1,H,W,C] */
  int32_t pt_back;         /* zero frames behind the end of x (the non-causal family: symmetric padding, and one frame
                            * behind the end for the stride-2 time downsample, model_3dnoncausal.py:80,86-87) */
  int32_t res_pool_off;    /* res_mode 3 avg-pool window: frames 2t-1+off .. 2t+1+off (1: non-causal, zero frame behind the end) */
} vt_conv_ex;
int32_t vt_op_conv_ex(int32_t precision, const vt_conv_ex* e, const void* x, const void* cache, const float* w,
                      const float* bias, const void* res, const float* gamma, const float* beta, void* out, void* out2,
                      void* stream);
/* Encoder conv_out with the KL / FSQ regularizer applied in the convolution's epilogue (regularizers.py:82-92,153-178,
 * distributions.py:8-18): reg_mode 1 = KL (Co = 2*zc, zc in {4,8,16}; noise NULL = the mode), 2 = FSQ (Co = zc = len(levels)).
 * h_out (fp32 [B,Co,T,H,W]) may be NULL; z fp32 [B,zc,T,H,W]; indices int32 [B,T,H,W] (FSQ); kl_loss 1 float (KL).
 * vt_op_conv_regularize: v1.0 zero time padding.  vt_op_conv_regularize_ex: e carries the geometry (e->d) and the v1.1
 * time padding (t_mode, cacheT, with `cache` as in vt_op_conv_ex, and pt_back); its other fields are ignored. */
int32_t vt_op_conv_regularize(int32_t precision, const vt_conv_desc* d, const void* x, const float* w, const float* bias,
                              int32_t reg_mode, int32_t zc, const int32_t* fsq_levels, const float* noise, float* h_out,
                              float* z, int32_t* indices, float* kl_loss, void* stream);
int32_t vt_op_conv_regularize_ex(int32_t precision, const vt_conv_ex* e, const void* x, const void* cache, const float* w,
                                 const float* bias, int32_t reg_mode, int32_t zc, const int32_t* fsq_levels, const float* noise,
                                 float* h_out, float* z, int32_t* indices, float* kl_loss, void* stream);
/* A convolution followed by ReLU, as the LPIPS stack runs it (BF16 / EXACT_TC; d->res_mode must be 0).  Operands as vt_op_conv. */
int32_t vt_op_conv_relu(int32_t precision, const vt_conv_desc* d, const void* x, const float* w, const float* bias, void* out,
                        void* stream);
/* 2x2 / stride-2 max-pool (floor) of channels-last x [N,H,W,C] -> y [N,H/2,W/2,C] in the precision's activation type (bf16, or
 * hi|lo split rows compared as hi + lo); C % 8 == 0. */
int32_t vt_op_maxpool2x2(int32_t precision, const void* x, void* y, int64_t N, int32_t H, int32_t W, int32_t C, void* stream);
/* Encoder stem from the caller's fp32 [B,Ci,T,H,W] (t_rep replicated leading frames, two zero frames in front); out
 * channels-last [B,T+t_rep,H,W,Co] in the precision's activation type (BF16 / EXACT_TC). */
int32_t vt_op_conv_stem(int32_t precision, const float* x, const float* w, const float* bias, void* out, int32_t B,
                        int32_t Ci, int32_t T, int32_t H, int32_t W, int32_t Co, int32_t t_rep, void* stream);
/* The same with pt zero frames in front: 2 (causal, = vt_op_conv_stem) or 1 (the non-causal family: one zero frame at
 * each end, t_rep 0). */
int32_t vt_op_conv_stem_ex(int32_t precision, const float* x, const float* w, const float* bias, void* out, int32_t B,
                           int32_t Ci, int32_t T, int32_t H, int32_t W, int32_t Co, int32_t t_rep, int32_t pt, void* stream);
/* Decoder head of the BF16 mode (tap-planes GEMM + gather): x bf16 [B,T,H,W,Ci] -> out fp32 [B,Co,T-to_off,H,W]. */
int32_t vt_op_head_planes(const void* x, const float* w, const float* bias, float* out, int32_t B, int32_t T, int32_t H,
                          int32_t W, int32_t Ci, int32_t Co, int32_t to_off, void* stream);
/* "nearest 2x upsample then conv" through the phase-collapsed weights (kind 0: Upsample, w [Co,Ci,3,3];
 * kind 1: v1.0 TimeUpsampleResCausal2x, w [C,C,3,3,3], alpha = sigmoid(mix_factor); kind 2: the non-causal
 * TimeUpsampleRes2x, the same with the 3x3x3 conv zero-padded by one frame on both sides, model_3dnoncausal.py:105-115);
 * gamma/beta/out2 optional: the following LayerNorm(+SiLU) fused into the phase convolutions. */
int32_t vt_op_upsample_conv(int32_t precision, int32_t kind, const void* x, const float* w, const float* bias, float alpha,
                            const float* gamma, const float* beta, int32_t ln_silu, void* out, void* out2, int32_t B,
                            int32_t T, int32_t H, int32_t W, int32_t Ci, int32_t Co, void* stream);
/* ResnetCausalBlock1D (model_3dcausal.py:427-499) as the BF16 mode runs it for 128 channels (one fused launch):
 * n1 = silu(LN1(x)) and x bf16 channels-last [B,T,H,W,C]; w1, w2 fp32 [C,C,3]; out = x + conv2(silu(LN2(conv1(n1))));
 * optional out2 = act(LN3(out)) (g3/be3/out2 may be NULL). */
int32_t vt_op_tblock(const void* n1, const void* x, const float* w1, const float* b1, const float* g2, const float* be2,
                     const float* w2, const float* b2, const float* g3, const float* be3, int32_t out_silu, void* out,
                     void* out2, int32_t B, int32_t T, int32_t H, int32_t W, int32_t C, void* stream);
/* vt_op_tblock continuing a video streamed chunk by chunk.  Caches: bf16 [B,2,H,W,C] (the layout the executor keeps for a
 * temporal block's conv1 / conv2): n1_cache = the block input frames t-2, t-1 before this chunk, h_cache = its
 * silu(LN2(conv1)) frames t-2, t-1.  Both inputs NULL: the video's first chunk (zero padding in front).  The outputs receive
 * the same two frames after this chunk and must not alias the inputs. */
int32_t vt_op_tblock_cached(const void* n1, const void* x, const float* w1, const float* b1, const float* g2, const float* be2,
                            const float* w2, const float* b2, const float* g3, const float* be3, int32_t out_silu, void* out,
                            void* out2, const void* n1_cache_in, const void* h_cache_in, void* n1_cache_out, void* h_cache_out,
                            int32_t B, int32_t T, int32_t H, int32_t W, int32_t C, void* stream);
/* y = silu?(norm(x)) over channels-last x [rows, C]; groupnorm variants take frame geometry. */
int32_t vt_op_layernorm(int32_t precision, const void* x, const float* gamma, const float* beta, void* y,
                        int64_t rows, int32_t C, int32_t apply_silu, void* stream);
int32_t vt_op_groupnorm(int32_t precision, const void* x, const float* gamma, const float* beta, void* y,
                        int64_t frames, int64_t positions_per_frame, int32_t C, int32_t per_position,
                        int32_t apply_silu, void* workspace, int64_t workspace_bytes, void* stream);
/* per-frame single-head attention core: q,k,v,o channels-last [frames, H, W, C] (tokens = H*W positions of a frame);
 * scale = C^-0.5.  vt_op_attention_hw runs what the model path runs for a frame of H x W, chosen from H, W and C alone:
 *   BF16 / EXACT_TC, tokens > 1024, C % 64 == 0, C <= 512: one fused kernel (online softmax, no tokens x tokens buffer);
 *     workspace: the output plus V^T, frames * C * (tokens + tokens rounded up to 8) * (2 bytes BF16, 4 EXACT_TC) + 2048;
 *   BF16 / EXACT_TC, tokens <= 1024, tokens % 64 == 0 and C % 64 == 0: wgmma GEMMs through a materialised score matrix;
 *   otherwise (and in FMA32): fp32 FMAs through a materialised score matrix.
 * vt_op_attention takes a token count and lays the tokens out as an image 8 wide (one row if tokens % 8 != 0): the same
 * arithmetic, not necessarily a model frame's tile plan.  workspace: frames*tokens*(8*tokens + 24*C) + 65536 bytes is
 * always enough. */
int32_t vt_op_attention(int32_t precision, const void* q, const void* k, const void* v, void* o, int32_t frames,
                        int32_t tokens, int32_t C, void* workspace, int64_t workspace_bytes, void* stream);
int32_t vt_op_attention_hw(int32_t precision, const void* q, const void* k, const void* v, void* o, int32_t frames,
                           int32_t H, int32_t W, int32_t C, void* workspace, int64_t workspace_bytes, void* stream);
int32_t vt_op_fsq(const float* h, int32_t d, const int32_t* levels, int64_t positions_per_batch, int32_t B,
                  float* codes, int32_t* indices, void* stream);
int32_t vt_op_fsq_indices_to_codes(const int32_t* indices, int32_t d, const int32_t* levels,
                                   int64_t positions_per_batch, int32_t B, float* codes, void* stream);
int32_t vt_op_kl(const float* h, const float* noise, int32_t zc, int64_t positions_per_batch, int32_t B, int32_t sample,
                 float* z, float* kl_loss, void* stream);

/* ---- FSQ auxiliary loss (FSQRegularizer.forward, regularizers.py:232-245): the clamped per-sample entropy, the codebook
 *      entropy of the batch-mean code distribution and the commitment MSE, computed from one small softmax per latent
 *      channel instead of the tokens x codebook distance matrix.  Two steps so that a caller can all-reduce the per-segment
 *      avg_prob between them (regularizers.py:49-59,240).  A segment is one untiled batch or one chunk of a tiled video.
 *      Supported: 1 <= d <= 8, every level >= 2, sum of the levels <= 256, codebook <= 2^22 codes (else VT_ERR_INVALID).
 *      Every reduction runs in a fixed order: repeated calls give the same bits. ---- */
/* workspace of vt_fsq_aux_partials for `tokens` = B * positions_per_batch tokens (-1 when unsupported) */
int64_t vt_fsq_aux_workspace_bytes(int32_t d, const int32_t* levels, int64_t tokens);
/* h: device fp32 [B,d,positions] (the encoder output before the FSQ bound; tokens in (b, t, h, w) order).  Outputs (device):
 * stats fp32 [2] = (per_sample_entropy, commit_loss), avg_prob fp32 [prod(levels)] = mean over the tokens of
 * softmax_j(2 * inv_temperature * <z, code_j>). */
int32_t vt_fsq_aux_partials(const float* h, int32_t d, const int32_t* levels, int64_t positions_per_batch, int32_t B,
                            float inv_temperature, float* stats, float* avg_prob, void* workspace, int64_t workspace_bytes,
                            void* stream);
/* stats [n_segments][2] and avg_prob [n_segments][J] as vt_fsq_aux_partials wrote them, avg_prob summed over world_size ranks
 * by the caller (world_size 1: not distributed).  Per segment: codebook_entropy over all J codes of avg_prob / world_size,
 * aux = (per_sample_entropy - diversity_gamma * codebook_entropy) * entropy_weight + commit_loss * commitment_weight.
 * aux_loss (1 float, device) = mean of the segments' aux; components (device, may be NULL) [n_segments][4] =
 * (per_sample_entropy, codebook_entropy, commit_loss, aux).  entropy_weight is calculate_entropy_loss_weight(n_steps). */
int32_t vt_fsq_aux_finalize(const float* stats, const float* avg_prob, int32_t n_segments, int32_t d, const int32_t* levels,
                            int32_t world_size, float entropy_weight, float diversity_gamma, float commitment_weight,
                            float* aux_loss, float* components, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VIDTOK_B200_H */
