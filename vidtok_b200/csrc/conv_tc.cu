// wgmma / TMA implicit-GEMM convolution for sm_90a (the tensor-core hot kernel).
//
// GEMM view of a causal convolution on channels-last activations [B,T,H,W,C]:
//   M = output positions, tiled as boxes of BT x BH x BW = 128 positions per CTA tile (two 64-row wgmma tiles),
//   N = Cout tile (BN in {32, 64, 128, 256}; fp32 accumulators in registers, BN / 2 per consumer thread and 64-row tile),
//   K = taps x Cin, consumed in steps of 64 channels (one 128-byte swizzle row) per tap.
// A operand, two formulations:
//   * halo mode (stride-1 kh x kw > 1 layers): ONE 5-D TMA box per (time tap, 64-channel chunk) loads the CTA tile's input
//     window with its spatial halo; the kh*kw taps are wgmma descriptors that start (bb*hP + c) 128-byte rows into it
//     (TcParams::halo).  ~3x fewer activation bytes cross L2 -> SM.
//   * otherwise one box {64, BW, BH, BT, 1} at (c0, w0+dw, h0+dh, t, b) per (tap, 64-channel chunk).
//   In both, spatial/temporal zero padding is the TMA out-of-bounds fill; the causal front pad is either skipped taps
//   (zeros), a clamped coordinate (replicate, v1.1 first chunk) or a second tensor map over the per-layer cache (v1.1
//   later chunks).  No im2col buffer, no padded copy.
// B operand: TMA box {64, BN} of the pre-packed K-major bf16 weights [Cout][taps*Cin].
// Both land in shared memory in the canonical K-major SWIZZLE_128B layout and feed wgmma.mma_async m64nBNk16.
// Warp roles (persistent CTA, one per SM): warps 0-7 = two consumer warpgroups (wgmma, then the epilogue straight from the
// accumulator registers: bias / residual / mix / LayerNorm / regularizer), warp 8 = TMA producer, which runs up to `stages`
// K steps ahead, across tile boundaries too, so that the next tile's operands load while the epilogue runs.  The bf16
// output tiles of the 256-channel schedule leave through shared memory: each warpgroup packs 64 rows x 64 channels at a
// time into its own swizzled staging buffer and one thread sends it with a bulk tensor store (TcParams::stage_out); all
// other outputs are stored per thread.
// The consumers follow one of two schedules (ping_pong()): cooperative, both warpgroups on every tile (rows
// [64 g, 64 g + 64)), or ping-pong, each warpgroup on every second tile (all 128 rows), their main loops taking turns so
// that one warpgroup's epilogue runs while the other one's MMAs issue.
#include <cuda.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <type_traits>

#include "common.cuh"
#include "kernels.h"
#include "tc_host.h"
#include "tc_ptx.cuh"

namespace vt {

namespace {

thread_local std::string g_tc_err;

struct TcParams {
  int B, To, Ho, Wo, Co, Ti;
  int BW, BH, BT;            // TMA box = BT x BH x BW positions = 128 rows
  int tilesW, tilesH, tilesT;
  int num_n_tiles, BN;
  long long num_tiles;
  int kt, kh, kw, Ci, num_kc;
  int st, pt, ph, pw, to_off;
  int sp;                    // spatial stride (1 or 2, same in H and W)
  int t_mode, cacheT;
  int stages;
  const float* bias;
  int res_mode;
  const bf16* res;
  long long rsB, rsT, rsH, rsW;
  int resT, res_t_mode, res_pool_off;
  const bf16* res_cache;
  float ra, rb;
  void* out;
  long long osB, osT, osH, osW, osC;
  int out_f32;               // 1: fp32 output with channel stride osC (external NCDHW heads), only n < Co_real stored
  int Co_real;
  int w_batched;             // weights differ per batch element (attention: K / V^T of each frame)
  // fused LayerNorm(+SiLU) over the output row (needs BN == Cout): 0 none, 1 out := act(LN(v)), 2 out := v and out2 := act(LN(v))
  int ln_mode, ln_silu;
  const float* ln_gamma;
  const float* ln_beta;
  void* out2;
  // residual add through the tensor pipe: BN/64 extra K steps with A = residual tile (TMA) and B = a slice of the
  // identity matrix, so `+ x` costs no epilogue work at all (res_mode 1 with ra == rb == 1)
  int res_mma;
  // halo mode (stride-1 spatial kernels): ONE TMA box per (time tap, 64-channel chunk) brings the input window of the
  // whole CTA tile plus its spatial halo ({64, hP, BH + kh - 1} rows of 128 B) into shared memory; the kh*kw spatial taps
  // are then wgmma descriptors that start (bb * hP + c) rows into that window, so the activation bytes pulled from L2
  // drop by ~kh*kw.  The CTA tile is 16 rows x 8 columns: an 8-row core group = 8 consecutive columns, group stride
  // (SBO) = hP rows, and hP % 8 == 0 keeps the swizzle phase of every group equal.
  int halo, hP, a_stages;
  uint32_t halo_bytes;
  // split operands (EXACT_TC mode, kernel template kSplit): activations and weights are stored as two fp16 planes
  // hi = fp16(v), lo = fp16(v - hi) side by side in the channel dimension ([..., hi(C) | lo(C)]); every K step loads
  // A_hi, A_lo, B_hi, B_lo and issues A_hi*B_hi + A_lo*B_hi + A_hi*B_lo into the same fp32 accumulator
  // (error ~2^-21 per product: fp32-class results on the 16-bit tensor pipe).  Channel coordinate of the lo plane:
  int split, a_lo, b_lo, o_lo;   // = Cin, Kpad, Cout
  float acc_scale;               // split: accumulator scale 2^-s of the pre-scaled weights
  // split, long K: the tensor core's fp32 accumulation is the dominant error there (it grows with the number of chained
  // MMAs), so the K steps of a tile are summed in `kparts` consecutive groups, each accumulated by the tensor core from
  // zero and added to a running fp32 sum with round-to-nearest (BN <= 128: the sum needs a second register set)
  int kparts;
  // regularizer epilogue on the fp32 heads (TcRegFusion): the row of a position is gathered in shared memory and the
  // thread that owns it holds every channel
  int reg_mode, reg_zc, reg_sample;
  const float* reg_noise;
  float* reg_z;
  int* reg_idx;
  double* reg_kl;
  FsqConst reg_fsq;
  uint32_t misc_off;         // byte offset of [bias | gamma | beta] x 2 (x 2 warpgroups in ping-pong) and the regularizer
                             // row buffer from the aligned base
  // bf16 outputs through shared memory: a warpgroup writes 64 rows x 64 channels of out (or out2) into its staging buffer
  // in the swizzled row layout and one bulk tensor store (maps o / o2) sends them, clipped at the tensor's edge.  The 64
  // rows are one half of the CTA tile: the box of the tile halved along dimension half_dim (1 w, 2 h, 3 t), half_ext long.
  int stage_out;             // the epilogue stores through the staging buffers
  uint32_t stage_smem;       // bytes of the staging buffers between the stage ring and the barriers (0: none in the plan)
  uint32_t stage_off;        // their byte offset from the aligned base
  int half_dim, half_ext;
  int relu;                  // ConvP::relu: a uniform flag, applied to the fp32 values before any store
};

struct TcMaps {
  CUtensorMap a[4];          // activation maps; [1..3] are the odd-parity views used by stride-2 convolutions
  CUtensorMap c;             // v1.1 causal cache
  CUtensorMap b;             // weights
  CUtensorMap r;             // residual tensor (output geometry), box = A box
  CUtensorMap e;             // 256 x 256 bf16 identity
  CUtensorMap o, o2;         // out / out2 (stage_out), box = 64 channels x one 64-row half of the CTA tile
};

constexpr int kConsumerWarps = 8;       // warps 0-7: two wgmma warpgroups
constexpr int kProducerWarp = kConsumerWarps;
// warps 8-11: the producer warpgroup (warp 8 issues the TMA loads); registers are allocated per warpgroup, so it hands
// most of its share to the consumers (setmaxnreg)
constexpr int kThreads = (kConsumerWarps + 4) * 32;
constexpr int kABytes = 128 * 128;      // 128 rows x 64 bf16
// consumer named barriers (0 is __syncthreads): 1 = bias buffer switch (cooperative), 2 = regularizer rows,
// kBarTurn + g = warpgroup g may start its next main loop, kBarBias + g = bias buffer switch of warpgroup g (ping-pong)
// kBarStage + g = staging buffer of warpgroup g written / free again
constexpr uint32_t kBarTurn = 3, kBarBias = 5, kBarStage = 7;
constexpr uint32_t kStageOutBytes = 64 * 128;   // staging buffer of one warpgroup: 64 rows x 64 bf16

// Ping-pong consumer schedule: with short K and a heavy epilogue (bf16 N tiles of 64 and 128 channels: 18-20 K steps
// against LayerNorm and one or two stored tiles) the cooperative schedule leaves the tensor pipe idle for the whole
// epilogue.  BN = 256 would need 256 accumulators per thread, the split operands a second register set for the K-group
// sum, and the BN = 32 regularizer heads gather each row across both warpgroups: those stay cooperative.
__host__ __device__ constexpr bool ping_pong(int BN, bool split) { return !split && (BN == 64 || BN == 128); }

using namespace tcx;

struct TileCoord {
  int b, t0, h0, w0, n0;
};
__device__ __forceinline__ TileCoord decode_tile(const TcParams& p, long long tile) {
  TileCoord c;
  const int nt = (int)(tile % p.num_n_tiles);
  long long m = tile / p.num_n_tiles;
  const int tw = (int)(m % p.tilesW); m /= p.tilesW;
  const int th = (int)(m % p.tilesH); m /= p.tilesH;
  const int tt = (int)(m % p.tilesT);
  c.b = (int)(m / p.tilesT);
  c.t0 = tt * p.BT; c.h0 = th * p.BH; c.w0 = tw * p.BW; c.n0 = nt * p.BN;
  return c;
}
// time coordinate of a tap for a tile; returns false when the whole box is causal zero padding (tap skipped)
__device__ __forceinline__ bool tap_time(const TcParams& p, const TileCoord& tc, int a, int& tv, bool& from_cache) {
  tv = (tc.t0 + p.to_off) * p.st + a - p.pt;
  from_cache = false;
  if (tv + p.BT <= 0) {
    if (p.t_mode == 0) return false;
    if (p.t_mode == 1) { tv = 0; return true; }
    from_cache = true;
    tv = p.cacheT + tv;
    return true;
  }
  return true;
}
// time taps of a tile that are loaded (not skipped as causal zero padding)
__device__ __forceinline__ int tile_taps(const TcParams& p, const TileCoord& tc) {
  int n = 0;
  for (int a = 0; a < p.kt; ++a) {
    int tv;
    bool from_cache;
    if (tap_time(p, tc, a, tv, from_cache)) ++n;
  }
  return n;
}

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// kStage: bf16 output tiles leave through the staging buffers (TcParams::stage_out); an instantiation of its own, so that
// neither way of storing holds registers for the other next to the accumulators
template <int BN, bool kSplit, bool kStage = false>
__global__ void __launch_bounds__(kThreads, 1)
conv_tc_kernel(const __grid_constant__ TcMaps maps, const TcParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t a_bytes = kABytes;
  constexpr uint32_t b_bytes = (uint32_t)BN * 128u;
  constexpr uint32_t kPl = kSplit ? 2u : 1u;               // operand planes per tile (hi | lo)
  // stage layout: [A_hi | A_lo | B_hi | B_lo] (A part absent in halo mode: the stage ring then holds B tiles only)
  const uint32_t stage_bytes = kPl * (p.halo ? b_bytes : a_bytes + b_bytes);
  const uint32_t win_bytes = kPl * p.halo_bytes;           // one halo window slot: [hi window | lo window]
  const uint32_t ring_base = smem_base + (p.halo ? (uint32_t)p.a_stages * win_bytes : 0u);
  // (the staging buffers of the bf16 output tiles lie between the ring and the barriers, 1024-byte aligned as every tile is)
  const uint32_t bar_base = ring_base + p.stages * stage_bytes + p.stage_smem;
  // barriers: full[stages], empty[stages], fullA[a_stages], emptyA[a_stages]
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (p.stages + s); };
  auto fullA_bar = [&](int s) { return bar_base + 8u * (2 * p.stages + s); };
  auto emptyA_bar = [&](int s) { return bar_base + 8u * (2 * p.stages + p.a_stages + s); };
  constexpr bool kPingPong = ping_pong(BN, kSplit);
  // [2][bias 256 | gamma 256 | beta 256], ping-pong: [2 warpgroups][2][...]
  float* sbias = reinterpret_cast<float*>(smem_gen + p.misc_off);
  float* rowbuf = sbias + 2 * 768;                                   // regularizer (BN 32, cooperative): [128 rows][33]

  if (threadIdx.x == 0) {
    // a stage / window is released by every consumer warp that reads it (both warpgroups, or the one that owns the tile in
    // ping-pong) once its own wait has seen the MMAs that read it complete (wgmma.wait_group tracks the executing warp's
    // share of the warpgroup's MMAs)
    constexpr uint32_t readers = kPingPong ? kConsumerWarps / 2 : kConsumerWarps;
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), readers);
    }
    for (int s = 0; s < p.a_stages; ++s) {
      mbar_init(fullA_bar(s), 1);
      mbar_init(emptyA_bar(s), readers);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int nsp = p.kh * p.kw;
  const int num_kc = p.num_kc, nstages = p.stages;
  const bool halo = p.halo != 0;
  const int res_steps = p.res_mma ? BN / 64 : 0;

  if (warp >= kProducerWarp) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp != kProducerWarp) return;
    // ===================== TMA producer =====================
    // The whole warp stays converged and elects one lane around the asynchronous instructions: addresses and
    // coordinates are warp-uniform values on the uniform datapath.
    const bool el = elect_one();
    if (el) {
      prefetch_tmap(&maps.a[0]);
      prefetch_tmap(&maps.b);
      if (p.sp == 2) { prefetch_tmap(&maps.a[1]); prefetch_tmap(&maps.a[2]); prefetch_tmap(&maps.a[3]); }
      if (p.t_mode == 2) prefetch_tmap(&maps.c);
      if (p.res_mma) { prefetch_tmap(&maps.r); prefetch_tmap(&maps.e); }
    }
    int stage = 0, sA = 0;
    uint32_t phase = 0, phA = 0;
    auto acquire = [&](uint32_t bytes) {
      mbar_wait(empty_bar(stage), phase ^ 1u);
      if (el) mbar_expect_tx(full_bar(stage), bytes);
    };
    auto advance = [&]() { if (++stage == nstages) { stage = 0; phase ^= 1u; } };
    // weight tile(s) of one K step into the B part of the current stage (split: hi plane, then lo plane at k + b_lo)
    auto load_b_planes = [&](uint32_t dst, const CUtensorMap* m, int kcol, int n, int wb_) {
      tma_load_3d(dst, m, full_bar(stage), kcol, n, wb_);
      if constexpr (kSplit) tma_load_3d(dst + b_bytes, m, full_bar(stage), p.b_lo + kcol, n, wb_);
    };
    // halo window of one (time tap, 64-channel chunk); lo_off = channel offset of the lo plane in that tensor
    auto load_window = [&](const CUtensorMap* m, int c0, int lo_off, int cw, int ch, int ct, int cb) {
      mbar_wait(emptyA_bar(sA), phA ^ 1u);
      if (el) {
        mbar_expect_tx(fullA_bar(sA), win_bytes);
        tma_load_5d(smem_base + (uint32_t)sA * win_bytes, m, fullA_bar(sA), c0, cw, ch, ct, cb);
        if constexpr (kSplit) tma_load_5d(smem_base + (uint32_t)sA * win_bytes + p.halo_bytes, m, fullA_bar(sA), lo_off + c0, cw, ch, ct, cb);
      }
      if (++sA == p.a_stages) { sA = 0; phA ^= 1u; }
    };
    for (long long tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const TileCoord tc = decode_tile(p, tile);
      const int wb = p.w_batched ? tc.b : 0;
      for (int a = 0; a < p.kt; ++a) {
        int tv;
        bool from_cache;
        if (!tap_time(p, tc, a, tv, from_cache)) continue;
        if (halo) {
          const CUtensorMap* mapA = from_cache ? &maps.c : &maps.a[0];
          for (int kc = 0; kc < num_kc; ++kc) {
            load_window(mapA, kc * 64, p.a_lo, tc.w0 - p.pw, tc.h0 - p.ph, tv, tc.b);
            int kcol = a * nsp * p.Ci + kc * 64;
            for (int sp = 0; sp < nsp; ++sp, kcol += p.Ci) {
              acquire(stage_bytes);
              if (el) load_b_planes(ring_base + stage * stage_bytes, &maps.b, kcol, tc.n0, wb);
              advance();
            }
          }
        } else {
          int kcol = a * nsp * p.Ci;
          for (int bb = 0; bb < p.kh; ++bb) {
            for (int c = 0; c < p.kw; ++c, kcol += p.Ci) {
              // input coordinates of the box origin.  Stride 2: tap (bb,c) reads rows 2*h + (bb-ph), i.e. row
              // h + ((bb-ph)>>1) of the parity-((bb-ph)&1) view (a tensor map over every second row/column)
              const int dh = bb - p.ph, dw2 = c - p.pw;
              int ch, cw;
              const CUtensorMap* mapA;
              if (p.sp == 2) {
                mapA = &maps.a[(dh & 1) * 2 + (dw2 & 1)];
                ch = tc.h0 + (dh >> 1);
                cw = tc.w0 + (dw2 >> 1);
              } else {
                mapA = &maps.a[0];
                ch = tc.h0 + dh;
                cw = tc.w0 + dw2;
              }
              if (from_cache) mapA = &maps.c;
              for (int kc = 0; kc < num_kc; ++kc) {
                acquire(stage_bytes);
                if (el) {
                  const uint32_t sa = smem_base + stage * stage_bytes;
                  tma_load_5d(sa, mapA, full_bar(stage), kc * 64, cw, ch, tv, tc.b);
                  if constexpr (kSplit) tma_load_5d(sa + a_bytes, mapA, full_bar(stage), p.a_lo + kc * 64, cw, ch, tv, tc.b);
                  load_b_planes(sa + kPl * a_bytes, &maps.b, kcol + kc * 64, tc.n0, wb);
                }
                advance();
              }
            }
          }
        }
      }
      // out += I * residual : A = residual tile of this output box, channels [n0 + 64g, +64); B = identity columns
      // (split: A_hi and A_lo tiles of the residual against the same identity tile; the B_lo slot stays unused)
      for (int g = 0; g < res_steps; ++g) {
        if (halo) {
          load_window(&maps.r, tc.n0 + g * 64, p.o_lo, tc.w0 - p.pw, tc.h0 - p.ph, tc.t0, tc.b);
          acquire(b_bytes);
          if (el) tma_load_3d(ring_base + stage * stage_bytes, &maps.e, full_bar(stage), g * 64, 0, 0);
        } else {
          acquire(kPl * a_bytes + b_bytes);
          if (el) {
            const uint32_t sa = smem_base + stage * stage_bytes;
            tma_load_5d(sa, &maps.r, full_bar(stage), tc.n0 + g * 64, tc.w0, tc.h0, tc.t0, tc.b);
            if constexpr (kSplit) tma_load_5d(sa + a_bytes, &maps.r, full_bar(stage), p.o_lo + tc.n0 + g * 64, tc.w0, tc.h0, tc.t0, tc.b);
            tma_load_3d(sa + kPl * a_bytes, &maps.e, full_bar(stage), g * 64, 0, 0);
          }
        }
        advance();
      }
    }
    return;
  }

  // ===================== consumers: wgmma main loop, then the epilogue from the accumulator registers =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  constexpr int R = BN / 2;                  // accumulator registers per thread and 64-row half of a tile
  constexpr int kHalves = kPingPong ? 2 : 1; // 64-row halves of a tile that one warpgroup computes
  constexpr bool kSum = kSplit && BN <= 128;  // running fp32 sum of the K groups (TcParams::kparts)
  const int g = warp >> 2, wq = warp & 3;
  const bool leader = lane == 0;
  const uint32_t hi_b = desc_hi(1024u);
  const uint32_t hi_a = halo ? desc_hi((uint32_t)p.hP * 128u) : hi_b;
  // A rows 64 .. 127 of a tile: 64 rows further into a dense tile, 8 window rows (h) further in halo mode
  const uint32_t a_half = halo ? 8u * (uint32_t)p.hP * 128u : 64u * 128u;
  const uint32_t a_row_off = kPingPong ? 0u : (uint32_t)g * a_half;   // first A row of this warpgroup
  const uint32_t a_pl = halo ? p.halo_bytes : a_bytes;        // hi plane -> lo plane (A)
  const uint32_t b_addr0 = halo ? ring_base : smem_base + kPl * a_bytes;
  float acc[kHalves][R];
  float sum[kSum ? R : 1];
  int stage = 0, sA = 0, sR = 0;
  uint32_t phase = 0, phA = 0;
  // resources read by the most recent committed MMA group, released once it has completed
  int pend_stage = -1;
  bool pend_win = false;
  auto release = [&]() {
    if (leader) {
      if (pend_stage >= 0) mbar_arrive(empty_bar(pend_stage));
      if (pend_win) mbar_arrive(emptyA_bar(sR));
    }
    if (pend_win && ++sR == p.a_stages) sR = 0;
    pend_stage = -1;
    pend_win = false;
  };
  // one K step (64 channels): this group's 64 A rows (ping-pong: both 64-row halves) at byte address a_addr (a window row),
  // or of the stage's A tile when a_from_stage, against the B tile of the current stage; split: hi*hi + lo*hi (+ hi*lo
  // unless `res`: the residual steps multiply by the identity, which has no lo plane)
  auto kstep = [&](bool a_from_stage, uint32_t a_addr, uint32_t scale, bool res, bool last_of_window) {
    mbar_wait(full_bar(stage), phase);
    if (a_from_stage) a_addr = smem_base + stage * stage_bytes + a_row_off;
    const uint32_t b_addr = b_addr0 + stage * stage_bytes;
    const uint32_t al = desc_lo(a_addr), bl = desc_lo(b_addr);
    wgmma_fence();
#pragma unroll
    for (uint32_t j = 0; j < 4u; ++j) {
      const uint64_t ah = desc(al + 2u * j, hi_a), bh = desc(bl + 2u * j, hi_b);
      wgmma_k16<BN, kSplit>(acc[0], ah, bh, j == 0 ? scale : 1u);
      if constexpr (kPingPong) wgmma_k16<BN, kSplit>(acc[1], desc(al + (a_half >> 4) + 2u * j, hi_a), bh, j == 0 ? scale : 1u);
      if constexpr (kSplit) {
        wgmma_k16<BN, kSplit>(acc[0], desc(al + (a_pl >> 4) + 2u * j, hi_a), bh, 1u);
        if (!res) wgmma_k16<BN, kSplit>(acc[0], ah, desc(bl + (b_bytes >> 4) + 2u * j, hi_b), 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();
    release();
    pend_stage = stage;
    pend_win = last_of_window;
    if (++stage == nstages) { stage = 0; phase ^= 1u; }
  };

  // this thread's rows: rbase and rbase + 8 (ping-pong: and rbase + 64, rbase + 72), columns 8j + cq, 8j + cq + 1
  const int rbase = (kPingPong ? 0 : 64 * g) + 16 * wq + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const bool res_direct = (p.res_mode == 1 && !p.res_mma);
  const bool store_a = (p.ln_mode != 1);
  const float inv_n = 1.0f / (float)BN;
  int last_n0 = -1;
  uint32_t cbuf = 1;                         // bias / gamma / beta buffer in use (toggled whenever n0 changes)

  // ping-pong: the CTA's tiles alternate between the warpgroups, `owner` is the one of the current tile
  int owner = 0;
  for (long long tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, owner ^= 1) {
    const TileCoord tc = decode_tile(p, tile);
    if constexpr (kPingPong) {
      if (owner != g) {
        // the other warpgroup's tile: step the ring counters past its K steps and halo windows
        const int taps = tile_taps(p, tc);
        stage += taps * nsp * num_kc + res_steps;
        if ((stage / nstages) & 1) phase ^= 1u;
        stage %= nstages;
        if (halo) {
          const int nw = taps * num_kc + res_steps;
          sA += nw;
          if ((sA / p.a_stages) & 1) phA ^= 1u;
          sA %= p.a_stages;
          sR = (sR + nw) % p.a_stages;
        }
        continue;
      }
      // the tensor pipe serves one main loop at a time: start once the other warpgroup has issued its previous tile
      if (tile != blockIdx.x) named_bar_sync(kBarTurn + g, kConsumerWarps * 32);
    }
    // ---- main loop
    uint32_t G = 0xFFFFFFFFu;                // K steps per group (kparts)
    if constexpr (kSum) {
      if (p.kparts > 1) {
        const uint32_t nk = (uint32_t)(tile_taps(p, tc) * nsp * num_kc + res_steps);
        G = (nk + (uint32_t)p.kparts - 1u) / (uint32_t)p.kparts;
      }
#pragma unroll
      for (int i = 0; i < R; ++i) sum[i] = 0.f;
    }
    uint32_t ks = 0, accum = 0;
    auto step = [&](bool a_from_stage, uint32_t a_addr, bool res, bool last_of_window) {
      if constexpr (kSum) {
        if (ks > 0 && ks % G == 0) {
          wgmma_wait<0>();
          acc_fence(acc[0]);
          release();
#pragma unroll
          for (int i = 0; i < R; ++i) sum[i] += acc[0][i];
          accum = 0;
        }
      }
      kstep(a_from_stage, a_addr, accum, res, last_of_window);
      accum = 1;
      ++ks;
    };
    for (int a = 0; a < p.kt; ++a) {
      int tv;
      bool from_cache;
      if (!tap_time(p, tc, a, tv, from_cache)) continue;
      if (halo) {
        for (int kc = 0; kc < num_kc; ++kc) {
          mbar_wait(fullA_bar(sA), phA);
          const uint32_t win = smem_base + (uint32_t)sA * win_bytes + a_row_off;
          for (int bb = 0; bb < p.kh; ++bb)
            for (int c = 0; c < p.kw; ++c)
              step(false, win + (uint32_t)(bb * p.hP + c) * 128u, false, bb == p.kh - 1 && c == p.kw - 1);
          if (++sA == p.a_stages) { sA = 0; phA ^= 1u; }
        }
      } else {
        for (int s = nsp * num_kc; s > 0; --s) step(true, 0u, false, false);
      }
    }
    for (int gr = 0; gr < res_steps; ++gr) {
      if (halo) {
        mbar_wait(fullA_bar(sA), phA);
        step(false, smem_base + (uint32_t)sA * win_bytes + a_row_off + (uint32_t)(p.ph * p.hP + p.pw) * 128u, true, true);
        if (++sA == p.a_stages) { sA = 0; phA ^= 1u; }
      } else {
        step(true, 0u, true, false);
      }
    }
    // the other warpgroup's next tile (the CTA's next one) may start issuing now
    if constexpr (kPingPong) {
      if (tile + gridDim.x < p.num_tiles) named_bar_arrive(kBarTurn + (g ^ 1), kConsumerWarps * 32);
    }
    wgmma_wait<0>();
#pragma unroll
    for (int hf = 0; hf < kHalves; ++hf) acc_fence(acc[hf]);
    release();
    if constexpr (kSum) {
#pragma unroll
      for (int i = 0; i < R; ++i) acc[0][i] += sum[i];
    }

    // ---- epilogue
    if (tc.n0 != last_n0) {
      // all warps of the consumers of a tile (both warpgroups, or one in ping-pong) walk the same tile sequence, so this
      // branch is uniform across them; a warp can only be one barrier behind, which is why two buffers are enough
      last_n0 = tc.n0;
      cbuf ^= 1u;
      constexpr int nthr = kPingPong ? 128 : kConsumerWarps * 32;
      float* b_ = sbias + ((kPingPong ? 2 * g : 0) + cbuf) * 768;
      for (int i = threadIdx.x % nthr; i < BN; i += nthr) {
        b_[i] = (p.bias && tc.n0 + i < p.Co_real) ? p.bias[tc.n0 + i] : 0.f;
        // with SiLU the bf16 normalisation produces y/2 directly (silu(y) = h + h*tanh(h), h = y/2)
        if (p.ln_mode) { const float sc = (p.ln_silu && !kSplit) ? 0.5f : 1.0f; b_[256 + i] = sc * p.ln_gamma[tc.n0 + i]; b_[512 + i] = sc * p.ln_beta[tc.n0 + i]; }
      }
      named_bar_sync(kPingPong ? kBarBias + g : 1u, nthr);
    }
    const float* bias_s = sbias + ((kPingPong ? 2 * g : 0) + cbuf) * 768;
    const float* gamma_s = bias_s + 256;
    const float* beta_s = bias_s + 512;

#pragma unroll
    for (int hf = 0; hf < kHalves; ++hf) {
      float (&acc_h)[R] = acc[hf];
      // first row of this half; opaque to the compiler, so that the address arithmetic of the second half is not hoisted
      // over the first half's epilogue, where it would hold registers that the accumulators of both halves need
      int row0 = rbase + 64 * hf;
      asm volatile("" : "+r"(row0));
      // geometry of this thread's two rows of this half
      bool valid[2];
      long long ooff[2];
      auto row_geom = [&](int row, int& t, int& h, int& w) {
        const int dw = halo ? (row & 7) : row % p.BW;
        const int dh = halo ? (row >> 3) : (row / p.BW) % p.BH;
        const int dt = halo ? 0 : row / (p.BW * p.BH);
        t = tc.t0 + dt; h = tc.h0 + dh; w = tc.w0 + dw;
        return (t < p.To) && (h < p.Ho) && (w < p.Wo);
      };
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        int t, h, w;
        valid[r] = row_geom(row0 + 8 * r, t, h, w);
        ooff[r] = (long long)tc.b * p.osB + (long long)t * p.osT + (long long)h * p.osH + (long long)w * p.osW;
      }
      // residual value of channel pair (c, c + 1) of a row: bf16 pair, or hi + lo fp16 pairs (split)
      auto res_pair = [&](const bf16* rp, int c, float& x0, float& x1) {
        const uint32_t hw = *reinterpret_cast<const uint32_t*>(rp + c);
        if constexpr (kSplit) {
          const uint32_t lw = *reinterpret_cast<const uint32_t*>(rp + p.o_lo + c);
          x0 = f16_lo(hw) + f16_lo(lw);
          x1 = f16_hi(hw) + f16_hi(lw);
        } else {
          x0 = bf16_lo(hw);
          x1 = bf16_hi(hw);
        }
      };
      // v = rb * (acc + bias) + ra * R, in place; the residual one row at a time, so that only that row's residual
      // pointers are live next to the accumulators
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + cq;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float f = kSplit ? fmaf(acc_h[4 * j + e], p.acc_scale, bias_s[c + (e & 1)]) : acc_h[4 * j + e] + bias_s[c + (e & 1)];
          if (p.rb != 1.0f) f *= p.rb;
          acc_h[4 * j + e] = f;
        }
      }
      if (res_direct || p.res_mode == 3) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          int t, h, w;
          if (!row_geom(row0 + 8 * r, t, h, w)) continue;
          const bf16* r0 = nullptr;
          const bf16* r1 = nullptr;
          const bf16* r2 = nullptr;
          if (res_direct) {
            r0 = p.res + (long long)tc.b * p.rsB + (long long)t * p.rsT + (long long)h * p.rsH + (long long)w * p.rsW + tc.n0;
          } else {
            // avg-pool of residual frames 2t-1, 2t, 2t+1 (front pad: zero / frame 0 / 1-frame cache)
            const long long sp = (long long)tc.b * p.rsB + (long long)h * p.rsH + (long long)w * p.rsW + tc.n0;
            const int ta = 2 * t - 1 + p.res_pool_off, tb = ta + 1, tcn = ta + 2;
            if (ta >= 0) r0 = p.res + sp + (long long)ta * p.rsT;
            else if (p.res_t_mode == 1) r0 = p.res + sp;
            else if (p.res_t_mode == 2) r0 = p.res_cache + (((long long)tc.b * p.Ho + h) * p.Wo + w) * (long long)p.Co * (kSplit ? 2 : 1) + tc.n0;
            if (tb < p.resT) r1 = p.res + sp + (long long)tb * p.rsT;
            if (tcn < p.resT) r2 = p.res + sp + (long long)tcn * p.rsT;
          }
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int c = 8 * j + cq;
            if (res_direct) {
              float x0, x1;
              res_pair(r0, c, x0, x1);
              acc_h[4 * j + 2 * r] = fmaf(p.ra, x0, acc_h[4 * j + 2 * r]);
              acc_h[4 * j + 2 * r + 1] = fmaf(p.ra, x1, acc_h[4 * j + 2 * r + 1]);
            } else {
              float s0 = 0.f, s1 = 0.f, x0, x1;
              if (r0) { res_pair(r0, c, x0, x1); s0 += x0; s1 += x1; }
              if (r1) { res_pair(r1, c, x0, x1); s0 += x0; s1 += x1; }
              if (r2) { res_pair(r2, c, x0, x1); s0 += x0; s1 += x1; }
              const float s3 = p.ra * (1.0f / 3.0f);
              acc_h[4 * j + 2 * r] = fmaf(s3, s0, acc_h[4 * j + 2 * r]);
              acc_h[4 * j + 2 * r + 1] = fmaf(s3, s1, acc_h[4 * j + 2 * r + 1]);
            }
          }
        }
      }
      if (p.relu) {
        // (v < 0 ? 0 : v keeps a NaN, as torch's ReLU does)
#pragma unroll
        for (int i = 0; i < R; ++i) acc_h[i] = acc_h[i] < 0.f ? 0.f : acc_h[i];
      }

      if (p.out_f32) {
        // external fp32 heads / attention scores: direct stores, only the real output channels
        if (p.out) {
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            if (!valid[r]) continue;
            float* of = reinterpret_cast<float*>(p.out) + ooff[r];
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int n = tc.n0 + 8 * j + cq + e;
                if (n < p.Co_real) of[(long long)n * p.osC] = acc_h[4 * j + 2 * r + e];
              }
          }
        }
        if (p.reg_mode) {
          // regularizer on the complete fp32 row of a position (heads with Cout <= 32: BN == 32, n0 == 0): the rows are
          // gathered in shared memory, thread i < 128 then owns row i with all of its channels
          if constexpr (BN == 32) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
              for (int e = 0; e < 4; ++e) rowbuf[(rbase + 8 * (e >> 1)) * 33 + 8 * j + cq + (e & 1)] = acc_h[4 * j + e];
            asm volatile("bar.sync 2, %0;" ::"n"(kConsumerWarps * 32) : "memory");
            if (threadIdx.x < 128) {
              const int row = threadIdx.x;
              float f[32];
#pragma unroll
              for (int c = 0; c < 32; ++c) f[c] = rowbuf[row * 33 + c];
              int t, h, w;
              const bool ok = row_geom(row, t, h, w);
              const long long plane = p.osC;                                  // T*H*W of the [B,C,T,H,W] tensors
              const long long pos = (long long)t * p.osT + (long long)h * p.osH + (long long)w * p.osW;
              if (p.reg_mode == 1) {
                float part = 0.f;
                // z_channels is a compile-time constant inside each case: f[] stays in registers (no dynamic indexing)
                auto kl_row = [&](auto ZC) {
                  constexpr int zc = decltype(ZC)::value;
                  const long long zb = (long long)tc.b * zc * plane + pos;
#pragma unroll
                  for (int c = 0; c < zc; ++c) {
                    float zv;
                    part += kl_sample_one(f[c], f[zc + c], p.reg_sample ? p.reg_noise[zb + c * plane] : 0.f, p.reg_sample, zv);
                    p.reg_z[zb + c * plane] = zv;
                  }
                };
                if (ok) {
                  if (p.reg_zc == 4) kl_row(std::integral_constant<int, 4>());
                  else if (p.reg_zc == 8) kl_row(std::integral_constant<int, 8>());
                  else kl_row(std::integral_constant<int, 16>());
                }
                double dsum = (double)part;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
                if (lane == 0) atomicAdd(p.reg_kl, dsum);
              } else if (ok) {
                const long long zb = (long long)tc.b * p.reg_zc * plane + pos;
                float idx = 0.f;
#pragma unroll
                for (int c = 0; c < VT_MAX_FSQ; ++c)
                  if (c < p.reg_zc) p.reg_z[zb + c * plane] = fsq_code(p.reg_fsq, c, f[c], idx);
                if (p.reg_idx) p.reg_idx[(long long)tc.b * plane + pos] = (int)idx;
              }
            }
            asm volatile("bar.sync 2, %0;" ::"n"(kConsumerWarps * 32) : "memory");
          }
        }
        continue;
      }

      if constexpr (kStage) {
        static_assert(!kSplit && BN == 256, "staged stores: the cooperative bf16 schedule");
        {
          // bf16 tiles through the warpgroup's staging buffer, 64 channels at a time.  The arithmetic is that of the
          // per-thread path below; packing the bf16-rounded values a second time reproduces the same words.
          float rstd[2], nmr[2];
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            float s = 0.f, q = 0.f;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
              const float f0 = acc_h[4 * j + 2 * r], f1 = acc_h[4 * j + 2 * r + 1];
              s += f0 + f1;
              q = fmaf(f0, f0, q);
              q = fmaf(f1, f1, q);
              const uint32_t kp = pack_bf16x2(f0, f1);
              acc_h[4 * j + 2 * r] = bf16_lo(kp);
              acc_h[4 * j + 2 * r + 1] = bf16_hi(kp);
            }
            const float mean = quad_sum(s) * inv_n;
            float var = fmaf(-mean, mean, quad_sum(q) * inv_n);
            var = var < 0.f ? 0.f : var;
            rstd[r] = rsqrtf(var + 1e-6f);
            nmr[r] = -mean * rstd[r];
          }
          // this thread's words of a 64-channel chunk: rows lrow and lrow + 8 of the half (the same swizzle phase, 1024
          // bytes apart), 16-byte unit u, bytes 2 cq .. 2 cq + 3 of it.  A warp's 32 words fall into 32 banks.
          // (addresses derived from the opaque row0, so that they are formed here and not carried through the main loop)
          const uint32_t sbuf = smem_base + p.stage_off + (uint32_t)(row0 >> 6) * kStageOutBytes;
          const uint32_t sw = sbuf + swz128_unit(row0 & 63, 0) + 2u * cq;
          auto put_s = [&](int r, int u, uint32_t word) {
            asm volatile("st.shared.b32 [%0], %1;" ::"r"((sw ^ ((uint32_t)u << 4)) + 1024u * r), "r"(word) : "memory");
          };
          const bool issuer = (threadIdx.x & 127) == 0;   // bulk groups belong to the thread that commits them
          // the previous store has read the buffer: the warpgroup may write it again
          auto reserve = [&]() {
            if (issuer) bulk_wait_read<0>();
            named_bar_sync(kBarStage + g, 128);
          };
          // every thread's words are visible to the async proxy: send chunk k of this half to m
          auto send = [&](const CUtensorMap* m, int k) {
            fence_async_smem();
            named_bar_sync(kBarStage + g, 128);
            if (issuer) {
              const int ho = g * p.half_ext;   // this warpgroup's half: its offset along half_dim
              tma_store_5d(m, sbuf, tc.n0 + 64 * k, tc.w0 + (p.half_dim == 1 ? ho : 0), tc.h0 + (p.half_dim == 2 ? ho : 0),
                           tc.t0 + (p.half_dim == 3 ? ho : 0), tc.b);
              bulk_commit();
            }
          };
          if (store_a) {
#pragma unroll
            for (int k = 0; k < BN / 64; ++k) {
              reserve();
#pragma unroll
              for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int u = 0; u < 8; ++u) put_s(r, u, pack_bf16x2(acc_h[4 * (8 * k + u) + 2 * r], acc_h[4 * (8 * k + u) + 2 * r + 1]));
              send(&maps.o, k);
            }
          }
          if (p.ln_mode) {
            const CUtensorMap* nmap = p.ln_mode == 1 ? &maps.o : &maps.o2;
#pragma unroll
            for (int k = 0; k < BN / 64; ++k) {
              reserve();
#pragma unroll
              for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                  const int j = 8 * k + u, c = 8 * j + cq;
                  float y0 = fmaf(fmaf(acc_h[4 * j + 2 * r], rstd[r], nmr[r]), gamma_s[c], beta_s[c]);
                  float y1 = fmaf(fmaf(acc_h[4 * j + 2 * r + 1], rstd[r], nmr[r]), gamma_s[c + 1], beta_s[c + 1]);
                  if (p.ln_silu) {
                    // y holds h = LN(v)/2 (gamma, beta were halved): silu = h + h * tanh(h)
                    y0 = fmaf(y0, tanh_approx(y0), y0);
                    y1 = fmaf(y1, tanh_approx(y1), y1);
                  }
                  put_s(r, u, pack_bf16x2(y0, y1));
                }
              send(nmap, k);
            }
          }
          continue;
        }
      }

      // 16-bit outputs: bf16 pairs, or hi | lo fp16 planes (split)
      auto put = [&](void* optr, int r, int c, float y0, float y1) {
        bf16* o = reinterpret_cast<bf16*>(optr) + ooff[r] + tc.n0 + c;
        if constexpr (kSplit) {
          const uint32_t hw = pack_f16x2(y0, y1);
          *reinterpret_cast<uint32_t*>(o) = hw;
          *reinterpret_cast<uint32_t*>(o + p.o_lo) = pack_f16x2(y0 - f16_lo(hw), y1 - f16_hi(hw));
        } else {
          *reinterpret_cast<uint32_t*>(o) = pack_bf16x2(y0, y1);
        }
      };
      if constexpr (kSplit) {
        // EXACT_TC: two-pass LayerNorm statistics on the fp32 values, full-precision SiLU
        if (store_a) {
#pragma unroll
          for (int r = 0; r < 2; ++r)
            if (valid[r])
#pragma unroll
              for (int j = 0; j < BN / 8; ++j) put(p.out, r, 8 * j + cq, acc_h[4 * j + 2 * r], acc_h[4 * j + 2 * r + 1]);
        }
        if (p.ln_mode) {
          void* nout = p.ln_mode == 1 ? p.out : p.out2;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            float s = 0.f;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) s += acc_h[4 * j + 2 * r] + acc_h[4 * j + 2 * r + 1];
            const float mean = quad_sum(s) * inv_n;
            float q = 0.f;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
              const float d0 = acc_h[4 * j + 2 * r] - mean, d1 = acc_h[4 * j + 2 * r + 1] - mean;
              q = fmaf(d0, d0, q);
              q = fmaf(d1, d1, q);
            }
            const float rstd = 1.0f / sqrtf(quad_sum(q) * inv_n + 1e-6f);
            if (!valid[r]) continue;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
              const int c = 8 * j + cq;
              float y0 = (acc_h[4 * j + 2 * r] - mean) * rstd * gamma_s[c] + beta_s[c];
              float y1 = (acc_h[4 * j + 2 * r + 1] - mean) * rstd * gamma_s[c + 1] + beta_s[c + 1];
              if (p.ln_silu) { y0 = silu_tc(y0); y1 = silu_tc(y1); }
              put(nout, r, c, y0, y1);
            }
          }
        }
      } else {
        // BF16: statistics from the fp32 values, the normalised values from their bf16 rounding (what the unfused
        // conv -> LayerNorm pair reads back from memory)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float s = 0.f, q = 0.f;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const float f0 = acc_h[4 * j + 2 * r], f1 = acc_h[4 * j + 2 * r + 1];
            s += f0 + f1;
            q = fmaf(f0, f0, q);
            q = fmaf(f1, f1, q);
            const uint32_t kp = pack_bf16x2(f0, f1);
            if (store_a && valid[r]) *reinterpret_cast<uint32_t*>(reinterpret_cast<bf16*>(p.out) + ooff[r] + tc.n0 + 8 * j + cq) = kp;
            acc_h[4 * j + 2 * r] = bf16_lo(kp);
            acc_h[4 * j + 2 * r + 1] = bf16_hi(kp);
          }
          if (!p.ln_mode) continue;
          // LayerNorm over the Cout values of this row (model_3dcausal.py:62-80, eps 1e-6), optional SiLU (:26-27)
          const float mean = quad_sum(s) * inv_n;
          float var = fmaf(-mean, mean, quad_sum(q) * inv_n);
          var = var < 0.f ? 0.f : var;
          const float rstd = rsqrtf(var + 1e-6f);
          const float nmr = -mean * rstd;
          if (!valid[r]) continue;
          void* nout = p.ln_mode == 1 ? p.out : p.out2;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int c = 8 * j + cq;
            float y0 = fmaf(fmaf(acc_h[4 * j + 2 * r], rstd, nmr), gamma_s[c], beta_s[c]);
            float y1 = fmaf(fmaf(acc_h[4 * j + 2 * r + 1], rstd, nmr), gamma_s[c + 1], beta_s[c + 1]);
            if (p.ln_silu) {
              // y holds h = LN(v)/2 (gamma, beta were halved): silu = h + h * tanh(h)
              y0 = fmaf(y0, tanh_approx(y0), y0);
              y1 = fmaf(y1, tanh_approx(y1), y1);
            }
            put(nout, r, c, y0, y1);
          }
        }
      }
    }
  }
  // the last bulk stores of this warpgroup have read its staging buffer, and are complete, before the CTA can exit
  if (kStage && (threadIdx.x & 127) == 0) bulk_wait<0>();
}

// 256 x 256 diagonal matrix `value` * I (bf16, or fp16 for the split mode)
__global__ void fill_identity_kernel(bf16* e, int f16, float value) {
  const int r = blockIdx.x, c = threadIdx.x;
  if (f16) reinterpret_cast<__half*>(e)[r * 256 + c] = __float2half_rn(r == c ? value : 0.0f);
  else e[r * 256 + c] = __float2bfloat16_rn(r == c ? value : 0.0f);
}

// ---------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------
bool choose_tile(const ConvP& p, int rows, int& BW, int& BH, int& BT) {
  const bool allow_bt = (p.st == 1) && (p.t_mode == 0);
  long long best = -1;
  auto ceil_to = [](int v, int b) { return (long long)((v + b - 1) / b) * b; };
  for (int bw = 128; bw >= 8; bw >>= 1) {
    for (int bh = rows / bw; bh >= 1; bh >>= 1) {
      if (bh > 256) continue;
      const int bt = rows / (bw * bh);
      if (bt > 1 && !allow_bt) continue;
      if (bt > 16) continue;
      const long long padded = ceil_to(p.Wo, bw) * ceil_to(p.Ho, bh) * ceil_to(p.To, bt);
      // prefer less padding; then square-ish spatial tiles (halo reuse in L2); then BT == 1
      const long long cost = padded * 1024 + (long long)(bw > 16 ? bw - 16 : 16 - bw) * 4 + (bt - 1);
      if (best < 0 || cost < best) { best = cost; BW = bw; BH = bh; BT = bt; }
    }
  }
  return best >= 0;
}
// N tile: the widest wgmma instantiation (32, 64, 128, 256) that divides Cout
int choose_bn(int Co) {
  for (int bn = 256; bn >= 32; bn >>= 1)
    if (Co % bn == 0) return bn;
  return 0;
}

// The residual-through-MMA identity of device dev: 256 x 256 bf16 I, or the 16 fp16 matrices 2^s * I of the split mode.
// Made once per device and precision, and filled (s synchronised) before any launch can read it.  Making it allocates and
// synchronises, which a capturing stream must not do: there it is an error (vt_model_finalize makes both in advance).
cudaError_t identity_tiles(int dev, bool split, cudaStream_t s, const bf16** out) {
  static bf16* ident_dev[2][kMaxDevices] = {{nullptr}};
  static std::mutex ident_mu;
  const int ik = split ? 1 : 0;
  std::lock_guard<std::mutex> lock(ident_mu);
  if (!ident_dev[ik][dev]) {
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(s, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone) {
      cudaGetLastError();
      g_tc_err = "the residual identity tiles do not exist yet and the stream is capturing";
      return cudaErrorStreamCaptureUnsupported;
    }
    const int nmat = split ? 16 : 1;
    bf16* e = nullptr;
    cudaError_t err = cudaMalloc(&e, (size_t)nmat * 256 * 256 * sizeof(bf16));
    if (err != cudaSuccess) { g_tc_err = "cudaMalloc(identity)"; return err; }
    for (int i = 0; i < nmat; ++i) fill_identity_kernel<<<256, 256, 0, s>>>(e + (size_t)i * 256 * 256, ik, ldexpf(1.0f, i));
    if ((err = cudaStreamSynchronize(s)) != cudaSuccess) { cudaFree(e); g_tc_err = "identity fill"; return err; }
    ident_dev[ik][dev] = e;
  }
  *out = ident_dev[ik][dev];
  return cudaSuccess;
}

}  // namespace

const char* conv_tc_last_error() { return g_tc_err.c_str(); }

cudaError_t conv_tc_prepare_identity(cudaStream_t s) {
  int dev = 0;
  if (cudaError_t e = current_device(dev)) return e;
  const bf16* unused;
  for (int split = 0; split < 2; ++split)
    if (cudaError_t e = identity_tiles(dev, split != 0, s, &unused)) return e;
  return cudaSuccess;
}

bool conv_tc_plan(const ConvP& p, DType tout, const TcLnFusion* ln, const TcRegFusion* reg, int w_batches, TcPlan* out) {
  g_tc_err.clear();
  auto no = [&](const char* why) { g_tc_err = why; return false; };
  if (p.Ci % 64 != 0) return no("Cin % 64 != 0");
  const int Co_pad = (p.Co + 31) / 32 * 32;
  if (choose_bn(Co_pad) == 0) return no("Cout has no valid N tile");
  const bool split = p.split != 0;
  const long long cw = split ? 2 : 1;   // bf16 elements per logical channel (hi | lo planes)
  if (split ? (tout == DT_BF16) : (tout == DT_SPLIT)) return no("activation layout of input and output differ");
  if (p.isC != 1 || p.isW != cw * p.Ci || p.isH != (long long)p.Wi * cw * p.Ci || p.isT != (long long)p.Hi * p.Wi * cw * p.Ci) return no("input is not dense channels-last");
  if (p.isB % 8 != 0) return no("batch stride not 16-byte aligned");
  if (tout != DT_F32) {
    if (p.Co % 32 != 0) return no("bf16 output needs Cout % 32 == 0");
    if (p.osC != 1 || p.osW % 8 != 0 || p.osH % 8 != 0 || p.osT % 8 != 0 || p.osB % 8 != 0) return no("output rows are not 16-byte aligned channels-last");
  }
  if (!((p.sh == 1 && p.sw == 1) || (p.sh == 2 && p.sw == 2))) return no("spatial stride");
  if (p.sh == 2 && ((p.Hi | p.Wi) & 1)) return no("stride-2 needs even H, W");
  if (p.st != 1 && p.st != 2) return no("time stride");
  if (p.ut != 1 || p.uh != 1 || p.uw != 1 || p.t_rep != 0) return no("folded upsampling / replicate prefix");
  if (p.res_mode != 0 && p.res_mode != 1 && p.res_mode != 3) return no("residual mode");
  if (p.res_mode != 0 && tout == DT_F32) return no("residual with fp32 output");
  if (p.t_mode == 2 && p.sh != 1) return no("cache mode with spatial stride");
  if (p.Wi > 65535 || p.Hi > 65535) return no("extent");
  if (w_batches > 1 && w_batches != p.B) return no("batched weights need one weight matrix per batch element");
  if (p.relu && ((ln && ln->mode) || (reg && reg->mode))) return no("ReLU with a fused LayerNorm or regularizer epilogue");
  TcPlan t = TcPlan();
  t.p = p; t.tout = tout; t.w_batches = w_batches;
  const int nk = p.kt * p.kh * p.kw * (p.Ci / 64);   // K steps
  // A fused LayerNorm needs one N tile over Cout.  Split mode: N tiles wider than 128 have no registers left for the running
  // sum of the kparts groups, and from 16 K steps on, where the plan sums in kparts, the tensor core's chained fp32
  // accumulation alone would exceed fp32-class error (measured 1.2-1.4x the 4e-5 (1 + |ref|) bound at 72-108 K steps, 256
  // channels), so such a LayerNorm runs as its own kernel after a kparts convolution.
  if (ln && ln->mode) {
    if (tout != DT_F32 && p.Co <= 256 && choose_bn(p.Co) == p.Co && (!split || p.Co <= 128 || nk < 16)) t.ln = *ln;
    else g_tc_err = "fused LayerNorm needs one N tile covering Cout, a 16-bit output and (split) Cout <= 128 or < 16 K steps";
  }
  // the regularizer epilogue: the thread that owns a position holds all of its channels (Co_pad == 32: one 32-wide N tile)
  if (reg && reg->mode) {
    const int need = reg->mode == 1 ? 2 * reg->zc : reg->zc;
    const bool zc_ok = reg->mode == 1 ? (reg->zc == 4 || reg->zc == 8 || reg->zc == 16) : reg->zc <= VT_MAX_FSQ;
    if (tout == DT_F32 && Co_pad == 32 && need <= p.Co && zc_ok && p.osW == 1) t.reg = *reg;
    else g_tc_err = "regularizer epilogue needs an fp32 [B,C,T,H,W] head with Cout <= 32 holding all latent channels";
  }
  // Tile geometry + shared-memory plan.  Split operands double every operand tile: when the halo windows leave fewer
  // than 2 pipeline stages, fall back to one A box per tap.
  auto plan = [&](bool allow_halo, int bn_cap) -> int {
    t.halo = 0; t.hP = 0; t.a_stages = 0; t.halo_bytes = 0;
    t.BN = choose_bn(Co_pad);
    if (bn_cap && t.BN > bn_cap) t.BN = bn_cap;
    if (!choose_tile(p, 128, t.BW, t.BH, t.BT)) { g_tc_err = "no tile shape"; return -1; }
    // halo mode: spatial taps reuse one shared-memory window (see TcParams::halo)
    const bool geom = p.sh == 1 && p.sw == 1 && p.kh * p.kw > 1 && p.kh <= 3 && p.kw <= 3 && p.Ho == p.Hi && p.Wo == p.Wi &&
                      w_batches <= 1 && p.Wo % 8 == 0 && p.Ho % 16 == 0;
    if (allow_halo && geom) {
      t.halo = 1;
      t.BW = 8; t.BH = 16; t.BT = 1;
      t.hP = 16;
      t.halo_bytes = (uint32_t)((16 + p.kh - 1) * t.hP * 128);
      t.a_stages = 2;
    }
    const size_t stage_bytes = (size_t)cw * ((t.halo ? 0 : (size_t)kABytes) + (size_t)t.BN * 128);
    const size_t budget = 225 * 1024;
    const size_t a_ring = (size_t)t.a_stages * t.halo_bytes * cw;
    // two bias / gamma / beta buffers per consumer group (ping-pong: one group per warpgroup), regularizer rows
    const size_t misc = (ping_pong(t.BN, split) ? 4 : 2) * 768 * 4 + (t.reg.mode ? 128 * 33 * 4 : 0);
    const size_t fixed = 1024 /*align*/ + misc + 16;
    if (budget < fixed + a_ring + 2 * (stage_bytes + 16)) return 1;
    int stages = (int)((budget - fixed - a_ring) / (stage_bytes + 16));
    if (stages > 8) stages = 8;
    // VT_TC_STAGES caps the pipeline depth: lets the tests run the shortest (2-stage) ring
    static const int cap = [] { const char* e = getenv("VT_TC_STAGES"); return e ? atoi(e) : 0; }();
    if (cap >= 2 && stages > cap) stages = cap;
    t.stages = stages;
    // smem layout from the 1024-aligned base:
    //   [halo windows] [stages x (A | B)] [staging buffers] [barriers] [bias/gamma/beta | regularizer rows]
    const size_t bars = 8 * (2 * (size_t)stages + 2 * (size_t)t.a_stages);
    // bf16 output tiles of the cooperative 256-channel schedule leave through one staging buffer per warpgroup
    // (TcParams::stage_out) where the two fit next to the ring as planned above: the ring's depth is never traded for
    // them, and the budget above leaves 2 KB of the SM's 227 KB for this.  Not in ping-pong: there the epilogue already
    // runs under the other warpgroup's MMAs, and the staged one measured slower (DESIGN.md section 8).
    const size_t staging = 2 * (size_t)kStageOutBytes;
    const bool staged = !split && tout == DT_BF16 && t.BN == 256 &&
                        1024 + ((a_ring + stages * stage_bytes + staging + bars + 15) & ~(size_t)15) + misc <= 227 * 1024;
    t.stage_out = staged ? 1 : 0;
    t.misc_off = (uint32_t)((a_ring + stages * stage_bytes + (staged ? staging : 0) + bars + 15) & ~(size_t)15);
    t.smem = 1024 + t.misc_off + misc;
    // split + long K: the K steps of a tile are summed in groups (TcParams::kparts; needs BN <= 128)
    t.kparts = (split && t.BN <= 128 && nk >= 16) ? (nk >= 64 ? 8 : 4) : 1;
    return 0;
  };
  // split + long K without a fused LayerNorm: narrow N tiles leave registers for the running sum (TcParams::kparts)
  const bool need_row = t.ln.mode != 0;
  const int bn_pref = (split && !need_row && w_batches <= 1) ? (nk >= 128 ? 64 : (nk >= 16 ? 128 : 0)) : 0;
  int rc = plan(true, bn_pref);
  if (rc == 1) rc = plan(false, bn_pref);
  if (rc == 1 && !need_row) rc = plan(false, 128);
  if (rc == 1) return no("not enough shared memory for 2 stages");
  if (rc != 0) return false;
  // (split mode: the weights carry a power-of-two scale 2^s that the epilogue removes from the whole accumulator, so the
  // residual is multiplied by 2^s * I -- exact in fp16 for s <= 15; larger scales fall back to the epilogue add)
  bool ident_ok = true;
  if (split) {
    const float ws = p.acc_scale != 0.f ? 1.0f / p.acc_scale : 1.0f;
    t.ident_s = ilogbf(ws);
    ident_ok = t.ident_s >= 0 && t.ident_s <= 15 && ldexpf(1.0f, t.ident_s) == ws;
  }
  t.res_mma = (ident_ok && p.res_mode == 1 && p.ra == 1.0f && p.rb == 1.0f && t.BN % 64 == 0 && p.Co % 64 == 0 && p.rsW % 8 == 0 &&
               p.rsH % 8 == 0 && p.rsT % 8 == 0 && p.rsB % 8 == 0 && (((uintptr_t)p.res) & 15) == 0) ? 1 : 0;
  *out = t;
  return true;
}

// (Co_pad = roundup(Co, 32): weight rows >= Co are zero)
cudaError_t launch_conv_tc(const TcPlan& pl, const bf16* x, const bf16* w_nk, void* out, cudaStream_t s, long long w_batch_stride) {
  if (!tmap_encoder()) { g_tc_err = "cuTensorMapEncodeTiled unavailable"; return cudaErrorNotSupported; }
  const ConvP& p = pl.p;
  const TcRegFusion& reg = pl.reg;
  const bool split = p.split != 0;
  const int cw = split ? 2 : 1;
  if (reg.mode ? (!reg.z || (reg.mode == 1 && (!reg.kl_acc || (reg.sample && !reg.noise)))) : !out) { g_tc_err = "null output"; return cudaErrorInvalidValue; }
  if (p.t_mode == 2 && (!p.cache || p.cacheT <= 0)) { g_tc_err = "cache mode without cache"; return cudaErrorInvalidValue; }
  int dev = 0;
  const cudaError_t dev_err = current_device(dev);
  if (dev_err != cudaSuccess) { g_tc_err = "no current device, or its index is out of range"; return dev_err; }
  const int Co_pad = (p.Co + 31) / 32 * 32, Kpad = p.kt * p.kh * p.kw * p.Ci;
  TcParams t;
  memset(&t, 0, sizeof(t));
  t.BW = pl.BW; t.BH = pl.BH; t.BT = pl.BT; t.BN = pl.BN;
  t.halo = pl.halo; t.hP = pl.hP; t.a_stages = pl.a_stages; t.halo_bytes = pl.halo_bytes;
  t.stages = pl.stages; t.misc_off = pl.misc_off; t.kparts = pl.kparts; t.res_mma = pl.res_mma;
  // a bulk tensor store needs a 16-byte aligned tensor, which the per-thread stores do not
  t.stage_smem = pl.stage_out ? 2 * kStageOutBytes : 0;
  t.stage_off = (uint32_t)pl.a_stages * pl.halo_bytes + (uint32_t)pl.stages * (uint32_t)((pl.halo ? 0 : kABytes) + pl.BN * 128);
  t.stage_out = (pl.stage_out && ((uintptr_t)out & 15) == 0 && ((uintptr_t)pl.ln.out2 & 15) == 0) ? 1 : 0;
  t.tilesW = (p.Wo + t.BW - 1) / t.BW; t.tilesH = (p.Ho + t.BH - 1) / t.BH; t.tilesT = (p.To + t.BT - 1) / t.BT;
  t.num_n_tiles = Co_pad / t.BN;
  t.num_tiles = (long long)p.B * t.tilesT * t.tilesH * t.tilesW * t.num_n_tiles;
  t.split = split ? 1 : 0; t.a_lo = p.Ci; t.b_lo = Kpad; t.o_lo = pl.o_lo ? pl.o_lo : p.Co;
  t.acc_scale = (split && p.acc_scale != 0.f) ? p.acc_scale : 1.0f;
  t.B = p.B; t.To = p.To; t.Ho = p.Ho; t.Wo = p.Wo; t.Co = p.Co; t.Ti = p.Ti;
  t.kt = p.kt; t.kh = p.kh; t.kw = p.kw; t.Ci = p.Ci; t.num_kc = p.Ci / 64;
  t.st = p.st; t.pt = p.pt; t.ph = p.ph; t.pw = p.pw; t.to_off = p.to_off; t.sp = p.sh;
  t.t_mode = p.t_mode; t.cacheT = p.cacheT;
  t.bias = p.bias; t.res_mode = p.res_mode; t.res = (const bf16*)p.res;
  t.rsB = p.rsB; t.rsT = p.rsT; t.rsH = p.rsH; t.rsW = p.rsW; t.resT = p.resT; t.res_t_mode = p.res_t_mode; t.res_pool_off = p.res_pool_off;
  t.res_cache = (const bf16*)p.res_cache; t.ra = p.ra; t.rb = p.rb;
  t.out = out; t.osB = p.osB; t.osT = p.osT; t.osH = p.osH; t.osW = p.osW; t.osC = p.osC;
  t.out_f32 = (pl.tout == DT_F32) ? 1 : 0;
  t.Co_real = p.Co;
  t.ln_mode = pl.ln.mode; t.ln_silu = pl.ln.silu ? 1 : 0; t.ln_gamma = pl.ln.gamma; t.ln_beta = pl.ln.beta; t.out2 = pl.ln.out2;
  if (reg.mode) {
    t.reg_mode = reg.mode; t.reg_zc = reg.zc; t.reg_sample = reg.sample; t.reg_noise = reg.noise; t.reg_z = reg.z;
    t.reg_idx = reg.indices; t.reg_kl = reg.kl_acc;
    if (reg.mode == 2) t.reg_fsq = make_fsq_const(reg.zc, reg.fsq_levels);
  }
  t.w_batched = pl.w_batches > 1 ? 1 : 0;
  t.relu = p.relu ? 1 : 0;

  TcMaps maps;
  // activation view: element (c, w, h, t, b) at base + c + w*sw_ + h*sh_ + t*isT + b*bs  (elements)
  auto encode_act = [&](CUtensorMap* m, const bf16* base, int Wn, int Hn, long long sw_, long long sh_, int Tn, long long st_, long long bs) -> bool {
    cuuint64_t dims[5] = {(cuuint64_t)(cw * p.Ci), (cuuint64_t)Wn, (cuuint64_t)Hn, (cuuint64_t)Tn, (cuuint64_t)p.B};
    cuuint64_t strides[4] = {(cuuint64_t)sw_ * 2, (cuuint64_t)sh_ * 2, (cuuint64_t)st_ * 2, (cuuint64_t)bs * 2};
    cuuint32_t box[5] = {64, (cuuint32_t)t.BW, (cuuint32_t)t.BH, (cuuint32_t)t.BT, 1};
    if (t.halo) { box[1] = (cuuint32_t)t.hP; box[2] = (cuuint32_t)(16 + p.kh - 1); }
    return encode_tmap_16b(m, 5, base, dims, strides, box, "activation", g_tc_err);
  };
  if (p.sh == 1) {
    if (!encode_act(&maps.a[0], x, p.Wi, p.Hi, p.isW, p.isH, p.Ti, p.isT, p.isB)) return cudaErrorInvalidValue;
    maps.a[1] = maps.a[2] = maps.a[3] = maps.a[0];
  } else {
    // parity views: rows hp, hp+2, ... and columns wp, wp+2, ...
    for (int hp = 0; hp < 2; ++hp)
      for (int wp = 0; wp < 2; ++wp)
        if (!encode_act(&maps.a[hp * 2 + wp], x + (long long)hp * p.isH + (long long)wp * p.isW, (p.Wi - wp + 1) / 2,
                        (p.Hi - hp + 1) / 2, 2 * p.isW, 2 * p.isH, p.Ti, p.isT, p.isB))
          return cudaErrorInvalidValue;
  }
  if (p.t_mode == 2) {
    if (!encode_act(&maps.c, (const bf16*)p.cache, p.Wi, p.Hi, p.isW, p.isH, p.cacheT, p.isT, (long long)p.cacheT * p.Hi * p.Wi * p.Ci * cw)) return cudaErrorInvalidValue;
  } else {
    maps.c = maps.a[0];
  }
  {
    const int nb = pl.w_batches > 1 ? pl.w_batches : 1;
    // split weights: [Co_pad][hi(Kpad) | lo(Kpad)]
    cuuint64_t dims[3] = {(cuuint64_t)(cw * Kpad), (cuuint64_t)Co_pad, (cuuint64_t)nb};
    cuuint64_t strides[2] = {(cuuint64_t)(cw * Kpad) * 2, (cuuint64_t)(nb > 1 ? w_batch_stride : (long long)cw * Kpad * Co_pad) * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)t.BN, 1};
    if (!encode_tmap_16b(&maps.b, 3, w_nk, dims, strides, box, "weights", g_tc_err)) return cudaErrorInvalidValue;
  }
  // output / residual maps (output geometry) and the identity used by the residual-through-MMA K steps
  auto encode_out = [&](CUtensorMap* m, const void* base, int Tn, long long sW, long long sH, long long sT, long long sB, int bw, int bh, int bt) -> bool {
    cuuint64_t dims[5] = {(cuuint64_t)(cw * p.Co), (cuuint64_t)p.Wo, (cuuint64_t)p.Ho, (cuuint64_t)Tn, (cuuint64_t)p.B};
    cuuint64_t strides[4] = {(cuuint64_t)sW * 2, (cuuint64_t)sH * 2, (cuuint64_t)sT * 2, (cuuint64_t)sB * 2};
    cuuint32_t box[5] = {64, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bt, 1};
    return encode_tmap_16b(m, 5, base, dims, strides, box, "output/residual", g_tc_err);
  };
  maps.r = maps.a[0]; maps.e = maps.b;
  if (t.res_mma) {
    const bf16* ident = nullptr;
    if (cudaError_t err = identity_tiles(dev, split, s, &ident)) return err;
    ident += (size_t)pl.ident_s * 256 * 256;
    if (!encode_out(&maps.r, p.res, p.resT, p.rsW, p.rsH, p.rsT, p.rsB, t.halo ? t.hP : t.BW, t.halo ? 16 + p.kh - 1 : t.BH, t.BT)) return cudaErrorInvalidValue;
    cuuint64_t dims[3] = {256, 256, 1};
    cuuint64_t strides[2] = {512, 256 * 512};
    cuuint32_t box[3] = {64, (cuuint32_t)t.BN, 1};
    if (!encode_tmap_16b(&maps.e, 3, ident, dims, strides, box, "identity", g_tc_err)) return cudaErrorInvalidValue;
  }
  if (t.stage_out) {
    // one 64-row half of the CTA tile: its box halved along the outermost dimension that is longer than one position
    int hb[3] = {t.BW, t.BH, t.BT};
    t.half_dim = t.BT > 1 ? 3 : (t.BH > 1 ? 2 : 1);
    t.half_ext = (hb[t.half_dim - 1] /= 2);
    if (!encode_out(&maps.o, out, p.To, p.osW, p.osH, p.osT, p.osB, hb[0], hb[1], hb[2])) return cudaErrorInvalidValue;
    maps.o2 = maps.o;
    if (t.ln_mode == 2 && !encode_out(&maps.o2, t.out2, p.To, p.osW, p.osH, p.osT, p.osB, hb[0], hb[1], hb[2])) return cudaErrorInvalidValue;
  } else {
    maps.o = maps.o2 = maps.a[0];
  }
  {
    static SmemLimitOnce smem_limit;
    cudaError_t e = smem_limit.ensure(dev, 227 * 1024, conv_tc_kernel<32, false>, conv_tc_kernel<64, false>, conv_tc_kernel<128, false>,
                                      conv_tc_kernel<256, false>, conv_tc_kernel<32, true>, conv_tc_kernel<64, true>,
                                      conv_tc_kernel<128, true>, conv_tc_kernel<256, true>, conv_tc_kernel<256, false, true>);
    if (e != cudaSuccess) { g_tc_err = "cudaFuncSetAttribute(smem)"; return e; }
  }
  const int num_sms = device_sms(dev);
  const unsigned grid = (unsigned)(t.num_tiles < num_sms ? t.num_tiles : num_sms);
  const double Mrows = (double)p.B * p.To * p.Ho * p.Wo;
  // plan key of the launch (profiler detail): geometry, tile, N tile, halo windows, fused LayerNorm, residual mode (m: through
  // the MMA), kparts, time padding (t0 zeros / t1 replicate / t2 cache) and pipeline stages; " pad<front>.<back>" only when
  // the time padding is not the causal one (the non-causal family), " pool<off>" only for a shifted avg-pool window of
  // res_mode 3 and " relu" only when ReLU is on, so the keys of every other plan stay as they were
  char det[192] = "";
  if (prof_enabled()) {
    char pad[48] = "";
    const int pt_back = time_pad_back(p);
    int n = 0;
    if (p.pt != (p.kt - 1) + (1 - p.st) || pt_back != 0) n = snprintf(pad, sizeof(pad), " pad%d.%d", p.pt, pt_back);
    if (p.res_mode == 3 && p.res_pool_off != 0) snprintf(pad + n, sizeof(pad) - n, " pool%d", p.res_pool_off);
    snprintf(det, sizeof(det), "k%d%d%d s%d%d %d->%d @%dx%dx%d tile%dx%dx%d bn%d%s ln%d r%d%s p%d t%d st%d%s%s", p.kt, p.kh, p.kw, p.st, p.sh, p.Ci, p.Co, p.To, p.Ho, p.Wo, t.BT, t.BH, t.BW, t.BN, t.halo ? " halo" : "", t.ln_mode, p.res_mode, t.res_mma ? "m" : "", split ? t.kparts : 1, p.t_mode, t.stages, pad, p.relu ? " relu" : "");
  }
  ProfScope _ps(split ? "conv_tc3" : "conv_tc", 2.0 * Mrows * p.kt * p.kh * p.kw * p.Ci * p.Co,
                2.0 * cw * ((double)p.B * p.Ti * p.Hi * p.Wi * p.Ci) + Mrows * p.Co * (pl.tout == DT_F32 ? 4.0 : 2.0 * cw), s, det);
  auto launch = [&](auto kern) { kern<<<grid, kThreads, pl.smem, s>>>(maps, t); };
  if (t.stage_out) launch(conv_tc_kernel<256, false, true>);
  else switch (t.BN * 2 + (split ? 1 : 0)) {
    case 64: launch(conv_tc_kernel<32, false>); break;
    case 65: launch(conv_tc_kernel<32, true>); break;
    case 128: launch(conv_tc_kernel<64, false>); break;
    case 129: launch(conv_tc_kernel<64, true>); break;
    case 256: launch(conv_tc_kernel<128, false>); break;
    case 257: launch(conv_tc_kernel<128, true>); break;
    case 512: launch(conv_tc_kernel<256, false>); break;
    default: launch(conv_tc_kernel<256, true>); break;
  }
  count_launch();
  return cudaGetLastError();
}

}  // namespace vt
