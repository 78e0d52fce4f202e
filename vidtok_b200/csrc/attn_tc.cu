// Fused per-frame attention on wgmma (AttnBlockWrapper's core, vidtok/modules/model_3dcausal.py:129-141):
//   O = softmax(Q K^T / sqrt(C)) V        for every frame of channels-last q, k, v [frames, tokens, C]
// without the tokens x tokens score matrix: scores live in registers one 64 x 128 tile at a time, with a running row
// maximum and sum (online softmax, fp32, the scale folded into exp2).
//
// A CTA owns 64 query rows of one frame and walks the frame's KV tokens in tiles of 128, in order.  Warp roles: warps 0-7
// are two consumer warpgroups, warp 8 is the TMA producer (its warpgroup hands its registers to the consumers).  Per tile:
//   S   warpgroup g computes S[:, 64g .. 64g+63] = Q K[tile rows]^T over all C channels (Q resident in shared memory, K
//       streamed in 64-channel chunks through the stage ring)
//   row statistics: both warpgroups exchange their row maxima through shared memory; each writes its half of
//       P = exp2((S - m) log2(e) / sqrt(C)) once, in the canonical K-major SWIZZLE_128B layout, and its row sums
//   PV  warpgroup g owns a channel slice of O (up to 128 channels): O[:, slice] = alpha O[:, slice] + P V[tile rows, slice],
//       with V^T chunks streamed through the same ring
// Above 256 channels the KV walk runs once per 256-channel slice of O (passes), recomputing S: see kNC below.
// Positions past `tokens` are masked (-inf scores) and never stored; TMA zero-fills the reads past the end of a frame, and
// a 3-D tensor map [frames][tokens][channels] keeps every tile inside its frame.
//
// Split (EXACT_TC) operands: q, k, v rows are hi|lo fp16 planes; both products run hi*hi + lo*hi + hi*lo, P is split into
// hi|lo fp16 planes (scaled by 2^15 so that the lo plane of small probabilities stays in fp16's normal range), and each KV
// tile's P V is accumulated from zero and added to the running O in fp32 registers with round-to-nearest, so the tensor
// core's chained accumulation never spans more than one tile (as the kparts path of conv_tc).
//
// Determinism: a frame's output depends on its own q, k, v and on (tokens, C) only -- fixed KV order, no atomics, no split
// of the KV loop across CTAs, fixed-order sums of the two warpgroups' partial row sums.
//
// Workspace (the caller's): V^T, one transposed copy of v ([frames][C (x2 planes)][tokens rounded up to 8]), the size of v.
#include <cuda.h>

#include <cstdio>
#include <cstring>
#include <string>

#include "common.cuh"
#include "kernels.h"
#include "tc_host.h"
#include "tc_ptx.cuh"

namespace vt {

namespace {
using namespace tcx;

thread_local std::string g_at_err;
constexpr int kBM = 64;                   // query rows per CTA
constexpr int kBN = 128;                  // KV tokens per tile (64 per consumer warpgroup in S)
constexpr int kConsumerWarps = 8;
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kThreadsAt = (kConsumerWarps + 4) * 32;
constexpr uint32_t kTile = 64 * 128;      // 64 rows x 64 16-bit elements (8 KB)
constexpr uint32_t kUnit = 2 * kTile;     // one ring unit: a K chunk [128 tokens x 64 ch] or a V^T chunk [64 ch x 128 tokens]
constexpr float kPScale = 32768.0f;       // split P: 2^15 * p <= 32768 stays in fp16's range

struct AtParams {
  int tokens, C, nc;                      // nc = C / 64 channel chunks
  int passes;                             // O is computed in passes of 2 kNC chunks (S recomputed in each)
  int q_tiles, kv_tiles, stages;
  float sl2;                              // log2(e) / sqrt(C)
  bf16* o;                                // [frames][tokens][cw * C]
};
struct AtMaps {
  CUtensorMap q, k, vt;
};

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// smem layout from the 1024-aligned base:
//   [Q: cw * nc tiles][P: cw * 2 tiles][ring: stages x cw units][barriers: full, empty, q][row max | row sum: 2 x 2 x 64]
// kNC: O chunks per warpgroup and pass, the register arrays' size.  A pass computes 2 kNC chunks of O, the first kNC in
// warpgroup 0, the rest in warpgroup 1; C = 512 runs two passes of 256 channels (the S tile, 128 accumulators of a 256-
// channel slice and the split mode's per-tile P V would not fit the 168 registers ptxas gives a thread of this CTA).
template <bool kSplit, int kNC>
__global__ void __launch_bounds__(kThreadsAt, 1) attn_tc_kernel(const __grid_constant__ AtMaps maps, const AtParams p) {
  constexpr int cw = kSplit ? 2 : 1;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t q_base = smem_base;
  const uint32_t p_base = q_base + (uint32_t)(cw * p.nc) * kTile;
  const uint32_t ring_base = p_base + (uint32_t)cw * 2u * kTile;
  const uint32_t stage_bytes = (uint32_t)cw * kUnit;
  const uint32_t bar_base = ring_base + (uint32_t)p.stages * stage_bytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (p.stages + s); };
  const uint32_t q_bar = bar_base + 16u * p.stages;
  float* red_max = reinterpret_cast<float*>(smem_gen + (bar_base - smem_base) + 16u * p.stages + 16u);   // [2 groups][64 rows]
  float* red_sum = red_max + 2 * kBM;

  const int frame = blockIdx.x / p.q_tiles;
  const int qt = blockIdx.x % p.q_tiles;
  if (threadIdx.x == 0) {
    // a stage is released by every consumer warp: after the MMAs that read it completed, or at once when its group does
    // not use it (the other group's V^T chunk)
    for (int s = 0; s < p.stages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kConsumerWarps); }
    mbar_init(q_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= kProducerWarp) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp != kProducerWarp) return;
    // ===================== TMA producer: Q once, then per KV tile the nc K chunks and the nc V^T chunks =====================
    const bool el = elect_one();
    if (el) {
      prefetch_tmap(&maps.q); prefetch_tmap(&maps.k); prefetch_tmap(&maps.vt);
      mbar_expect_tx(q_bar, (uint32_t)(cw * p.nc) * kTile);
      // split rows are [hi C | lo C]: chunk c of the row (hi chunks, then lo chunks) starts at element 64 c
      for (int c = 0; c < cw * p.nc; ++c) tma_load_3d(q_base + (uint32_t)c * kTile, &maps.q, q_bar, 64 * c, qt * kBM, frame);
    }
    int stage = 0;
    uint32_t phase = 0;
    auto acquire = [&]() {
      mbar_wait(empty_bar(stage), phase ^ 1u);
      if (el) mbar_expect_tx(full_bar(stage), stage_bytes);
    };
    auto advance = [&]() { if (++stage == p.stages) { stage = 0; phase ^= 1u; } };
    for (int pass = 0; pass < p.passes; ++pass)
      for (int t = 0; t < p.kv_tiles; ++t) {
        const int kv0 = t * kBN;
        for (int i = 0; i < p.nc; ++i) {
          acquire();
          if (el) {
            const uint32_t sa = ring_base + (uint32_t)stage * stage_bytes;
            tma_load_3d(sa, &maps.k, full_bar(stage), 64 * i, kv0, frame);
            if (kSplit) tma_load_3d(sa + kUnit, &maps.k, full_bar(stage), p.C + 64 * i, kv0, frame);
          }
          advance();
        }
        const int cb = pass * 2 * kNC, ce = min(p.nc, cb + 2 * kNC);
        for (int i = cb; i < ce; ++i) {
          acquire();
          if (el) {
            const uint32_t sa = ring_base + (uint32_t)stage * stage_bytes;
            for (int kb = 0; kb < 2; ++kb) {
              tma_load_3d(sa + (uint32_t)kb * kTile, &maps.vt, full_bar(stage), kv0 + 64 * kb, 64 * i, frame);
              if (kSplit) tma_load_3d(sa + kUnit + (uint32_t)kb * kTile, &maps.vt, full_bar(stage), kv0 + 64 * kb, p.C + 64 * i, frame);
            }
          }
          advance();
        }
      }
    return;
  }

  // ===================== consumers =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int g = warp >> 2, wq = warp & 3;
  const uint32_t hi = desc_hi(1024u);
  const int cq = 2 * (lane & 3);
  const int rloc = 16 * wq + (lane >> 2);    // this thread's rows of the tile: rloc and rloc + 8
  float o[kNC][32];
  float s[32];
  int stage = 0, pend_stage = -1;
  uint32_t phase = 0;
  auto release = [&]() {
    if (lane == 0 && pend_stage >= 0) mbar_arrive(empty_bar(pend_stage));
    pend_stage = -1;
  };
  auto advance = [&]() { if (++stage == p.stages) { stage = 0; phase ^= 1u; } };
  // the other group's V^T chunk: wait until it is loaded (so that the release counts for this fill), release it
  auto skip_unit = [&]() {
    mbar_wait(full_bar(stage), phase);
    if (lane == 0) mbar_arrive(empty_bar(stage));
    advance();
  };
  auto pair_sync = [&]() { named_bar_sync(1, kConsumerWarps * 32); };
  mbar_wait(q_bar, 0);

  for (int pass = 0; pass < p.passes; ++pass) {
    // this pass's O chunks: [cb, cb + pc), group 0 owns the first nc0 of them
    const int cb = pass * 2 * kNC, pc = min(2 * kNC, p.nc - cb), nc0 = min(kNC, pc);
    const int my_nc = g == 0 ? nc0 : pc - nc0;
#pragma unroll
    for (int c = 0; c < kNC; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    for (int t = 0; t < p.kv_tiles; ++t) {
      // ---- S: this group's 64 KV columns of the tile, over the nc channel chunks
      for (int i = 0; i < p.nc; ++i) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t sa = ring_base + (uint32_t)stage * stage_bytes;
        const uint32_t al = desc_lo(q_base + (uint32_t)i * kTile), bl = desc_lo(sa + (uint32_t)g * 64u * 128u);
        wgmma_fence();
#pragma unroll
        for (uint32_t j = 0; j < 4u; ++j) {
          const uint64_t ah = desc(al + 2u * j, hi), bh = desc(bl + 2u * j, hi);
          wgmma_k16<64, kSplit>(s, ah, bh, (i == 0 && j == 0) ? 0u : 1u);
          if constexpr (kSplit) {
            wgmma_k16<64, kSplit>(s, desc(al + (((uint32_t)p.nc * kTile) >> 4) + 2u * j, hi), bh, 1u);
            wgmma_k16<64, kSplit>(s, ah, desc(bl + (kUnit >> 4) + 2u * j, hi), 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        release();
        pend_stage = stage;
        advance();
      }
      wgmma_wait<0>();
      acc_fence(s);
#pragma unroll
      for (int c = 0; c < kNC; ++c) acc_fence(o[c]);
      release();

      // ---- row statistics.  One buffer of each suffices: a group rewrites red_max only after the second barrier of this
      // tile, which the other group reaches after reading it, and red_sum only after the next tile's first barrier.
      const int kvb = t * kBN + 64 * g;
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (kvb + 8 * j + cq + (e & 1) >= p.tokens) s[4 * j + e] = -INFINITY;
          mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * j + e]);
        }
      mx[0] = quad_max(mx[0]);
      mx[1] = quad_max(mx[1]);
      if ((lane & 3) == 0) { red_max[g * kBM + rloc] = mx[0]; red_max[g * kBM + rloc + 8] = mx[1]; }
      // both groups are past their PV of the previous tile (the wait above): P may be overwritten after this barrier
      pair_sync();
      float alpha[2], nms[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int row = rloc + 8 * r;
        const float m_new = fmaxf(m_run[r], fmaxf(red_max[row], red_max[kBM + row]));   // finite: every tile has a valid column
        alpha[r] = exp2f((m_run[r] - m_new) * p.sl2);
        m_run[r] = m_new;
        nms[r] = -m_new * p.sl2;
      }
      float sm[2] = {0.f, 0.f};
      uint8_t* pblk = smem_gen + (p_base - smem_base) + (uint32_t)g * kTile;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int cc = 8 * j + cq, u = cc >> 3;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float p0 = exp2f(fmaf(s[4 * j + 2 * r], p.sl2, nms[r]));
          const float p1 = exp2f(fmaf(s[4 * j + 2 * r + 1], p.sl2, nms[r]));
          sm[r] += p0 + p1;
          const int row = rloc + 8 * r;
          // canonical K-major SWIZZLE_128B: 16-byte unit u of row `row` lives at unit u ^ (row & 7)
          uint8_t* dst = pblk + row * 128 + ((u ^ (row & 7)) << 4) + (cc & 7) * 2;
          if constexpr (kSplit) {
            const float q0 = p0 * kPScale, q1 = p1 * kPScale;
            const uint32_t h = pack_f16x2(q0, q1);
            *reinterpret_cast<uint32_t*>(dst) = h;
            *reinterpret_cast<uint32_t*>(dst + 2 * kTile) = pack_f16x2(q0 - f16_lo(h), q1 - f16_hi(h));
          } else {
            *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(p0, p1);
          }
        }
      }
      sm[0] = quad_sum(sm[0]);
      sm[1] = quad_sum(sm[1]);
      if ((lane & 3) == 0) { red_sum[g * kBM + rloc] = sm[0]; red_sum[g * kBM + rloc + 8] = sm[1]; }
      fence_async_smem();
      pair_sync();
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int row = rloc + 8 * r;
        l_run[r] = fmaf(l_run[r], alpha[r], red_sum[row] + red_sum[kBM + row]);
      }

      // ---- PV: this group's O chunks += P V^T[chunk] over the tile's 128 tokens
      if constexpr (!kSplit) {
#pragma unroll
        for (int c = 0; c < kNC; ++c)
#pragma unroll
          for (int i = 0; i < 32; ++i) o[c][i] *= alpha[(i >> 1) & 1];
      }
      if (g == 1)
        for (int i = 0; i < nc0; ++i) skip_unit();
#pragma unroll
      for (int c = 0; c < kNC; ++c) {
        if (c >= my_nc) break;
        mbar_wait(full_bar(stage), phase);
        const uint32_t sa = ring_base + (uint32_t)stage * stage_bytes;
        if constexpr (kSplit) {
          float d[32];
          wgmma_fence();
#pragma unroll
          for (uint32_t j = 0; j < 8u; ++j) {
            const uint32_t al = desc_lo(p_base + (j >> 2) * kTile) + 2u * (j & 3u), bl = desc_lo(sa + (j >> 2) * kTile) + 2u * (j & 3u);
            wgmma_k16<64, true>(d, desc(al, hi), desc(bl, hi), j == 0 ? 0u : 1u);
            wgmma_k16<64, true>(d, desc(al + ((2u * kTile) >> 4), hi), desc(bl, hi), 1u);
            wgmma_k16<64, true>(d, desc(al, hi), desc(bl + (kUnit >> 4), hi), 1u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          acc_fence(d);
          pend_stage = stage;
          release();
#pragma unroll
          for (int i = 0; i < 32; ++i) o[c][i] = fmaf(o[c][i], alpha[(i >> 1) & 1], d[i]);
        } else {
          wgmma_fence();
#pragma unroll
          for (uint32_t j = 0; j < 8u; ++j) {
            const uint32_t al = desc_lo(p_base + (j >> 2) * kTile) + 2u * (j & 3u), bl = desc_lo(sa + (j >> 2) * kTile) + 2u * (j & 3u);
            wgmma_k16<64, false>(o[c], desc(al, hi), desc(bl, hi), 1u);
          }
          wgmma_commit();
          wgmma_wait<1>();
          release();
          pend_stage = stage;
        }
        advance();
      }
      if (g == 0)
        for (int i = nc0; i < pc; ++i) skip_unit();
    }
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < kNC; ++c) acc_fence(o[c]);
    release();

    // ---- epilogue: O / l, rows past the end of the frame are not stored
    const int ch0 = 64 * (cb + (g == 0 ? 0 : nc0));
    const long long rs = (long long)cw * p.C;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = qt * kBM + rloc + 8 * r;
      if (row >= p.tokens) continue;
      const float inv = (kSplit ? 1.0f / kPScale : 1.0f) / l_run[r];
      bf16* orow = p.o + ((long long)frame * p.tokens + row) * rs;
#pragma unroll
      for (int c = 0; c < kNC; ++c) {
        if (c >= my_nc) break;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int col = ch0 + 64 * c + 8 * j + cq;
          const float v0 = o[c][4 * j + 2 * r] * inv, v1 = o[c][4 * j + 2 * r + 1] * inv;
          if constexpr (kSplit) {
            const uint32_t h = pack_f16x2(v0, v1);
            *reinterpret_cast<uint32_t*>(orow + col) = h;
            *reinterpret_cast<uint32_t*>(orow + p.C + col) = pack_f16x2(v0 - f16_lo(h), v1 - f16_hi(h));
          } else {
            *reinterpret_cast<uint32_t*>(orow + col) = pack_bf16x2(v0, v1);
          }
        }
      }
    }
    }
  }

  // v [frames][tokens][cols] -> vt [frames][cols][tpad] (16-bit elements; cols = cw * C)
  __global__ void attn_vt_kernel(const uint16_t* __restrict__ v, uint16_t* __restrict__ vt, int frames, int tokens, int cols, int tpad) {
    __shared__ uint16_t tile[32][33];
    const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int f = blockIdx.z; f < frames; f += gridDim.z) {
      for (int k = threadIdx.y; k < 32; k += 8) {
        const int t = t0 + k, c = c0 + threadIdx.x;
        if (t < tokens && c < cols) tile[k][threadIdx.x] = v[((long long)f * tokens + t) * cols + c];
      }
      __syncthreads();
      for (int k = threadIdx.y; k < 32; k += 8) {
        const int c = c0 + k, t = t0 + threadIdx.x;
        if (c < cols && t < tokens) vt[((long long)f * cols + c) * tpad + t] = tile[threadIdx.x][k];
      }
      __syncthreads();
    }
  }

  constexpr size_t kSmemBudget = 227 * 1024;
  size_t at_fixed_smem(int nc, bool split) {
    const int cw = split ? 2 : 1;
    return 1024 + (size_t)(cw * nc + cw * 2) * kTile + 16 + 2 * 2 * kBM * sizeof(float);
  }
  int at_stages(int nc, bool split) {
    const size_t per = (size_t)(split ? 2 : 1) * kUnit + 16;
    const size_t fixed = at_fixed_smem(nc, split);
    if (fixed + 2 * per > kSmemBudget) return 0;
    const int st = (int)((kSmemBudget - fixed) / per);
    return st > 8 ? 8 : st;
  }

  template <bool kSplit>
  cudaError_t launch_nc(int knc, const AtMaps& maps, const AtParams& p, unsigned grid, size_t smem, cudaStream_t s) {
    if (knc == 1) attn_tc_kernel<kSplit, 1><<<grid, kThreadsAt, smem, s>>>(maps, p);
    else attn_tc_kernel<kSplit, 2><<<grid, kThreadsAt, smem, s>>>(maps, p);
    return cudaGetLastError();
  }
  }  // namespace

  const char* attn_tc_last_error() { return g_at_err.c_str(); }

  bool attn_tc_supported(long long frames, long long tokens, int C, bool split) {
    g_at_err.clear();
    if (frames <= 0 || tokens <= 0) { g_at_err = "empty"; return false; }
    if (C <= 0 || C % 64 != 0 || C > 512) { g_at_err = "C must be a multiple of 64, at most 512"; return false; }
    if (tokens > (1LL << 30)) { g_at_err = "too many tokens per frame"; return false; }
    if (frames * ((tokens + kBM - 1) / kBM) >= (1LL << 31)) { g_at_err = "grid too large"; return false; }
    if (at_stages(C / 64, split) < 2) { g_at_err = "shared memory"; return false; }
    return true;
  }

  size_t attn_tc_workspace(long long frames, long long tokens, int C, bool split) {
    const long long tpad = (tokens + 7) / 8 * 8;
    return (size_t)frames * (split ? 2 : 1) * C * tpad * sizeof(bf16);
  }

  cudaError_t launch_attn_tc(const bf16* q, const bf16* k, const bf16* v, bf16* o, int frames, int H, int W, int C, bool split,
                             void* ws, cudaStream_t s) {
    if (!tmap_encoder()) { g_at_err = "cuTensorMapEncodeTiled unavailable"; return cudaErrorNotSupported; }
    const long long tokens = (long long)H * W;
    if (!attn_tc_supported(frames, tokens, C, split)) return cudaErrorInvalidValue;
    const int cw = split ? 2 : 1;
    const long long tpad = (tokens + 7) / 8 * 8;
    const int cols = cw * C;
    bf16* vt = (bf16*)ws;
    {
      char det[96] = "";
      if (prof_enabled()) snprintf(det, sizeof(det), "@%dx%dx%d c%d", frames, H, W, C);
      ProfScope _ps("attn_vt", 0.0, 2.0 * 2.0 * frames * tokens * cols, s, det);
      const dim3 grid((unsigned)((tokens + 31) / 32), (unsigned)(cols / 32), (unsigned)(frames < 65535 ? frames : 65535));
      attn_vt_kernel<<<grid, dim3(32, 8), 0, s>>>((const uint16_t*)v, (uint16_t*)vt, frames, (int)tokens, cols, (int)tpad);
      count_launch();
      const cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) { g_at_err = "V transpose launch"; return e; }
    }
    AtMaps maps;
    for (int i = 0; i < 2; ++i) {
      // q / k: [frames][tokens][cw * C], boxes of 64 channels x 64 (q) / 128 (k) tokens
      cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)tokens, (cuuint64_t)frames};
      cuuint64_t strides[2] = {(cuuint64_t)cols * 2, (cuuint64_t)tokens * cols * 2};
      cuuint32_t box[3] = {64, (cuuint32_t)(i ? kBN : kBM), 1};
      if (!encode_tmap_16b(i ? &maps.k : &maps.q, 3, i ? k : q, dims, strides, box, "q/k", g_at_err)) return cudaErrorInvalidValue;
    }
    {
      // V^T: [frames][cw * C][tpad], boxes of 64 tokens x 64 channels
      cuuint64_t dims[3] = {(cuuint64_t)tokens, (cuuint64_t)cols, (cuuint64_t)frames};
      cuuint64_t strides[2] = {(cuuint64_t)tpad * 2, (cuuint64_t)tpad * cols * 2};
      cuuint32_t box[3] = {64, 64, 1};
      if (!encode_tmap_16b(&maps.vt, 3, vt, dims, strides, box, "v^T", g_at_err)) return cudaErrorInvalidValue;
    }
    AtParams p;
    memset(&p, 0, sizeof(p));
    p.tokens = (int)tokens; p.C = C; p.nc = C / 64;
    const int knc = p.nc > 2 ? 2 : 1;
    p.passes = (p.nc + 2 * knc - 1) / (2 * knc);
    p.q_tiles = (int)((tokens + kBM - 1) / kBM);
    p.kv_tiles = (int)((tokens + kBN - 1) / kBN);
    p.stages = at_stages(p.nc, split);
    p.sl2 = 1.4426950408889634f / sqrtf((float)C);
    p.o = o;
    const size_t smem = at_fixed_smem(p.nc, split) + (size_t)p.stages * ((size_t)cw * kUnit + 16);
    int dev = 0;
    const cudaError_t dev_err = current_device(dev);
    if (dev_err != cudaSuccess) { g_at_err = "no current device, or its index is out of range"; return dev_err; }
    {
      static SmemLimitOnce smem_limit;
      const cudaError_t e = smem_limit.ensure(dev, (int)kSmemBudget, attn_tc_kernel<false, 1>, attn_tc_kernel<false, 2>,
                                              attn_tc_kernel<true, 1>, attn_tc_kernel<true, 2>);
      if (e != cudaSuccess) { g_at_err = "cudaFuncSetAttribute(smem)"; return e; }
    }
  const unsigned grid = (unsigned)((long long)frames * p.q_tiles);
  const double tk = (double)tokens;
  char det[96] = "";
  if (prof_enabled()) snprintf(det, sizeof(det), "@%dx%dx%d c%d st%d pass%d", frames, H, W, C, p.stages, p.passes);
  // algorithmic FLOPs 4 tokens^2 C per frame (the passes' recomputed S not counted); bytes: q, k, v read and o written once
  ProfScope _ps(split ? "attn_tc3" : "attn_tc", 4.0 * frames * tk * tk * C, 4.0 * frames * tk * cols * 2.0, s, det);
  const cudaError_t e = split ? launch_nc<true>(knc, maps, p, grid, smem, s) : launch_nc<false>(knc, maps, p, grid, smem, s);
  count_launch();
  if (e != cudaSuccess) g_at_err = "attn_tc launch";
  return e;
}

}  // namespace vt
