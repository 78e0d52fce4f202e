// Fused temporal residual block on wgmma (BF16 mode):
//   ResnetCausalBlock1D  (vidtok/modules/model_3dcausal.py:427-499)
//     h   = conv1(n1)                      n1 = silu(LN1(x)) is produced by the previous stage's epilogue
//     out = x + conv2(silu(LN2(h)))        both convs are causal k=3 temporal convolutions (CausalConv1d, :144-159)
// as ONE kernel.  A k=3 temporal convolution is point-wise in space, so a CTA that owns a strip of 128 positions and walks
// the frames in order keeps LN2(h) in shared memory: HBM sees n1 and x in and out (+ the next stage's LN'd copy) out, and the
// intermediate h never leaves the SM.
//
// Per CTA (persistent over strips of BW x BH = 128 positions), for t = 0 .. T-1, each of the two consumer warpgroups on its
// 64 rows of the strip:
//   G1(t): acc = sum_a W1[a] . n1[t-2+a]          A (n1 frame) and B (W1 slice) tiles by TMA; fp32 accumulators in registers
//   E1(t): H[t mod 3] = bf16(silu(LN2(acc + b1)))  written by the warpgroup straight into the canonical K-major SWIZZLE_128B
//          layout (the layout a TMA load would have produced), then fence.proxy.async: the ring is the next A operand
//   G2(t): acc = sum_a W2[a] . H[t-2+a]            A = the shared-memory ring, B (W2 slice) by TMA
//   E2(t): out[t] = acc + b2 + x[t]; optionally out2[t] = act(LN_next(out[t])) for the next stage
//          x[t] comes by TMA into the ring slot of frame t-2 (free once G2(t)'s first tap is done), E2 overwrites it with
//          out[t], and one bulk tensor store per warpgroup writes it back; out2 is stored per thread
// Causal zero padding = skipped taps.
//
// Cached variant (kCache, a video streamed chunk by chunk): the taps in front of frame 0 read the previous chunk's last two
// n1 frames (G1) and the ring slots of frames -2, -1 are preloaded from its last two LN2(h) frames (G2), so a chunk computes
// exactly what the whole clip computes for those frames.  After its last frame each strip writes the chunk's last two n1 and
// LN2(h) frames as the next caches (for a one-frame chunk, part old cache and part new frame).  Without input caches (the
// first chunk) the taps in front of frame 0 are zero padding, as in the uncached kernel.  Cache layout: bf16 [B,2,H,W,128],
// the buffers the two-launch path keeps for conv1 / conv2.  Warp roles: warps 0-7 = two consumer warpgroups, warp 8 = TMA producer (its warpgroup
// hands its registers to the consumers through setmaxnreg).
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

thread_local std::string g_tb_err;
constexpr int kC = 128;                 // channels (Cin == Cout) this kernel is built for
constexpr int kKc = kC / 64;            // 64-channel K chunks per tap
constexpr uint32_t kTile = 128 * 128;   // one operand tile: 128 rows x 64 bf16
constexpr int kHSlots = 3;
constexpr int kConsumerWarps = 8;
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kThreadsTb = (kConsumerWarps + 4) * 32;

struct TbParams {
  int B, T, H, W;
  int BW, BH;                // strip box, BW * BH == 128
  int tilesW, tilesH;
  long long num_strips;
  int stages;
  const float* bias1;
  const float* bias2;
  const float* g2;           // LayerNorm between the convolutions (norm2), eps 1e-6
  const float* b2;
  int ln_out, ln_out_silu;   // additionally write out2 = act(LN(out)) (the next stage's first norm)
  const float* g3;
  const float* b3;
  const bf16* x;
  bf16* out;
  bf16* out2;
  // kCache only
  const bf16* n1;
  int cached_in;             // cn1_in / ch_in hold frames -2, -1 (else zero padding: the first chunk)
  const bf16* cn1_in;
  const bf16* ch_in;
  bf16* cn1_out;
  bf16* ch_out;
};
struct TbMaps {
  CUtensorMap n1, w1, w2, cn1;
  CUtensorMap x, out;   // 64-row boxes: one consumer warpgroup's half of a strip
};

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// smem layout from the 1024-aligned base:
//   [H ring: 3 slots x kKc tiles][stage ring: stages x (A tile | B tile)][barriers: full, empty, x][constants]
template <bool kCache>
__global__ void __launch_bounds__(kThreadsTb, 1) tblock_tc_kernel(const __grid_constant__ TbMaps maps, const TbParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t h_base = smem_base;
  const uint32_t ring_base = h_base + kHSlots * kKc * kTile;
  const uint32_t stage_bytes = 2u * kTile;
  const uint32_t bar_base = ring_base + (uint32_t)p.stages * stage_bytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (p.stages + s); };
  auto x_bar = [&](int g) { return bar_base + 16u * p.stages + 8u * g; };   // x[t] of consumer warpgroup g has landed
  float* cst = reinterpret_cast<float*>(smem_gen + (bar_base - smem_base) + 16u * p.stages + 16u);   // bias1 | g2 | b2 | bias2 | g3 | b3

  for (int i = threadIdx.x; i < kC; i += kThreadsTb) {
    cst[i] = p.bias1 ? p.bias1[i] : 0.f;
    // with SiLU the normalisation produces y/2 directly (silu(y) = h + h*tanh(h), h = y/2)
    cst[kC + i] = 0.5f * p.g2[i];
    cst[2 * kC + i] = 0.5f * p.b2[i];
    cst[3 * kC + i] = p.bias2 ? p.bias2[i] : 0.f;
    const float sc = p.ln_out_silu ? 0.5f : 1.0f;
    cst[4 * kC + i] = p.ln_out ? sc * p.g3[i] : 0.f;
    cst[5 * kC + i] = p.ln_out ? sc * p.b3[i] : 0.f;
  }
  if (threadIdx.x == 0) {
    // a stage is released by every consumer warp once its own wait has seen the MMAs that read it complete
    for (int s = 0; s < p.stages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kConsumerWarps); }
    for (int g = 0; g < 2; ++g) mbar_init(x_bar(g), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= kProducerWarp) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp != kProducerWarp) return;
    // ===================== TMA producer: per frame the G1 steps (n1 tile + W1 slice), then the G2 steps (W2 slice) =====
    const bool el = elect_one();
    if (el) { prefetch_tmap(&maps.n1); prefetch_tmap(&maps.w1); prefetch_tmap(&maps.w2); }
    const bool front = kCache && p.cached_in;   // taps in front of frame 0 read the caches
    int stage = 0;
    uint32_t phase = 0;
    auto acquire = [&](uint32_t bytes) {
      mbar_wait(empty_bar(stage), phase ^ 1u);
      if (el) mbar_expect_tx(full_bar(stage), bytes);
    };
    auto advance = [&]() { if (++stage == p.stages) { stage = 0; phase ^= 1u; } };
    for (long long strip = blockIdx.x; strip < p.num_strips; strip += gridDim.x) {
      const int tw = (int)(strip % p.tilesW);
      const int th = (int)((strip / p.tilesW) % p.tilesH);
      const int b = (int)(strip / ((long long)p.tilesW * p.tilesH));
      const int w0 = tw * p.BW, h0 = th * p.BH;
      for (int t = 0; t < p.T; ++t) {
        for (int a = 0; a < 3; ++a) {
          const int tv = t - 2 + a;
          if (tv < 0 && !front) continue;
          for (int kc = 0; kc < kKc; ++kc) {
            acquire(2u * kTile);
            if (el) {
              const uint32_t sa = ring_base + stage * stage_bytes;
              if (kCache && tv < 0) tma_load_5d(sa, &maps.cn1, full_bar(stage), kc * 64, w0, h0, tv + 2, b);
              else tma_load_5d(sa, &maps.n1, full_bar(stage), kc * 64, w0, h0, tv, b);
              tma_load_3d(sa + kTile, &maps.w1, full_bar(stage), a * kC + kc * 64, 0, 0);
            }
            advance();
          }
        }
        for (int a = 0; a < 3; ++a) {
          if (t - 2 + a < 0 && !front) continue;
          for (int kc = 0; kc < kKc; ++kc) {
            acquire(kTile);
            if (el) tma_load_3d(ring_base + stage * stage_bytes + kTile, &maps.w2, full_bar(stage), a * kC + kc * 64, 0, 0);
            advance();
          }
        }
      }
    }
    return;
  }

  // ===================== consumers =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int g = warp >> 2, wq = warp & 3;
  const uint32_t hi = desc_hi(1024u);
  float acc[kC / 2];
  int stage = 0, pend_stage = -1;
  uint32_t phase = 0, xphase = 0;
  auto release = [&]() {
    if (lane == 0 && pend_stage >= 0) mbar_arrive(empty_bar(pend_stage));
    pend_stage = -1;
  };
  // one K step (64 channels) of this warpgroup's 64 rows: A from the stage (G1) or from the H ring at h_addr (G2)
  auto kstep = [&](bool a_from_stage, uint32_t h_addr, uint32_t scale) {
    mbar_wait(full_bar(stage), phase);
    const uint32_t sa = ring_base + stage * stage_bytes;
    const uint32_t al = desc_lo(a_from_stage ? sa + (uint32_t)g * 64u * 128u : h_addr), bl = desc_lo(sa + kTile);
    wgmma_fence();
#pragma unroll
    for (uint32_t j = 0; j < 4u; ++j) wgmma_k16<kC, false>(acc, desc(al + 2u * j, hi), desc(bl + 2u * j, hi), j == 0 ? scale : 1u);
    wgmma_commit();
    wgmma_wait<1>();
    release();
    pend_stage = stage;
    if (++stage == p.stages) { stage = 0; phase ^= 1u; }
  };
  auto finish = [&]() {
    wgmma_wait<0>();
    acc_fence(acc);
    release();
  };
  auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory"); };
  const float* bias1 = cst;
  const float* g2 = cst + kC;
  const float* b2 = cst + 2 * kC;
  const float* bias2 = cst + 3 * kC;
  const float* g3 = cst + 4 * kC;
  const float* b3 = cst + 5 * kC;
  const int cq = 2 * (lane & 3);
  const int rbase = 64 * g + 16 * wq + (lane >> 2);   // this thread's rows: rbase and rbase + 8
  const bool front = kCache && p.cached_in;
  const int gtid = threadIdx.x & 127;
  // ring slot of frame tv >= -2
  auto slot_of = [&](int tv) { return h_base + (uint32_t)((tv + kHSlots) % kHSlots) * kKc * kTile; };
  // 16-byte unit (8 channels from c) of ring row `row` in the canonical K-major SWIZZLE_128B layout
  auto ring_unit = [&](uint32_t slot, int row, int c) {
    return reinterpret_cast<uint4*>(smem_gen + (slot - smem_base) + (c >> 6) * kTile + swz128_unit(row, (c & 63) >> 3));
  };

  for (long long strip = blockIdx.x; strip < p.num_strips; strip += gridDim.x) {
    const int tw = (int)(strip % p.tilesW);
    const int th = (int)((strip / p.tilesW) % p.tilesH);
    const int b = (int)(strip / ((long long)p.tilesW * p.tilesH));
    long long pos0[2];   // position index (b, t = 0, h, w) of this thread's rows
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = rbase + 8 * r;
      const int h = th * p.BH + row / p.BW, w = tw * p.BW + row % p.BW;
      pos0[r] = (((long long)b * p.T) * p.H + h) * p.W + w;
    }
    const long long frame = (long long)p.H * p.W;
    // position (b, h, w) of unit i of this warpgroup's 64 rows (16 units of 8 channels per row) in a [B,2,H,W,128] cache
    auto cache_pos = [&](int i, int j, int& row) {
      row = 64 * g + (i >> 4);
      const int h = th * p.BH + row / p.BW, w = tw * p.BW + row % p.BW;
      return ((((long long)b * 2 + j) * p.H + h) * p.W + w) * kC + (i & 15) * 8;
    };
    if (front) {
      // ring slots of frames -2, -1 := the LN2(h) cache
      if (gtid == 0) bulk_wait_read<0>();
      wg_sync();   // every warp of the group is done with the previous strip's ring
      for (int j = 0; j < 2; ++j)
        for (int i = gtid; i < 64 * 16; i += 128) {
          int row;
          const long long off = cache_pos(i, j, row);
          *ring_unit(slot_of(j - 2), row, (i & 15) * 8) = *reinterpret_cast<const uint4*>(p.ch_in + off);
        }
      fence_async_smem();
      wg_sync();
    }
    // E2(t) finds x[t] (this warpgroup's 64 rows, brought by TMA) in the ring slot of frame t-2, which G2(t) no longer
    // reads once its first tap is done, and leaves out[t] in its place for one bulk tensor store
    const int box_w = tw * p.BW + (64 * g) % p.BW, box_h = th * p.BH + (64 * g) / p.BW;
    auto x_load = [&](int t) {
      if (gtid != 0) return;
      const uint32_t dst = slot_of(t - 2) + (uint32_t)g * 64u * 128u;
      mbar_expect_tx(x_bar(g), (uint32_t)kKc * 64u * 128u);
      for (int kc = 0; kc < kKc; ++kc) tma_load_5d(dst + (uint32_t)kc * kTile, &maps.x, x_bar(g), kc * 64, box_w, box_h, t, b);
    };
    for (int t = 0; t < p.T; ++t) {
      // ---- G1(t)
      uint32_t scale = 0;
      for (int a = 0; a < 3; ++a) {
        if (t - 2 + a < 0 && !front) continue;
        for (int kc = 0; kc < kKc; ++kc) { kstep(true, 0u, scale); scale = 1; }
      }
      finish();
      // ---- E1(t): H[t mod 3] = bf16(silu(LN2(acc + b1))); statistics from fp32, normalisation of the bf16-rounded h
      if (gtid == 0) bulk_wait_read<0>();   // the slot written here held out[t-1] for a bulk store
      wg_sync();   // every warp of the group is past G2(t-1), which read the slot written here
      const uint32_t slot = h_base + (uint32_t)(t % kHSlots) * kKc * kTile;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float s = 0.f, q = 0.f;
#pragma unroll
        for (int j = 0; j < kC / 8; ++j) {
          const int c = 8 * j + cq;
          const float f0 = acc[4 * j + 2 * r] + bias1[c], f1 = acc[4 * j + 2 * r + 1] + bias1[c + 1];
          s += f0 + f1;
          q = fmaf(f0, f0, q);
          q = fmaf(f1, f1, q);
          const uint32_t kp = pack_bf16x2(f0, f1);
          acc[4 * j + 2 * r] = bf16_lo(kp);
          acc[4 * j + 2 * r + 1] = bf16_hi(kp);
        }
        const float mean = quad_sum(s) * (1.0f / kC);
        float var = fmaf(-mean, mean, quad_sum(q) * (1.0f / kC));
        var = var < 0.f ? 0.f : var;
        const float rstd = rsqrtf(var + 1e-6f);
        const float nmr = -mean * rstd;
        const int row = rbase + 8 * r;
        uint8_t* hslot = smem_gen + (slot - smem_base);
#pragma unroll
        for (int j = 0; j < kC / 8; ++j) {
          const int c = 8 * j + cq;
          float y0 = fmaf(fmaf(acc[4 * j + 2 * r], rstd, nmr), g2[c], b2[c]);
          float y1 = fmaf(fmaf(acc[4 * j + 2 * r + 1], rstd, nmr), g2[c + 1], b2[c + 1]);
          y0 = fmaf(y0, tanh_approx(y0), y0);
          y1 = fmaf(y1, tanh_approx(y1), y1);
          const int cc = c & 63;
          *reinterpret_cast<uint32_t*>(hslot + (c >> 6) * kTile + swz128_unit(row, cc >> 3) + (cc & 7) * 2) = pack_bf16x2(y0, y1);
        }
      }
      fence_async_smem();
      wg_sync();
      // ---- G2(t): A = this group's rows of the H ring
      const bool tap0 = t >= 2 || front;   // G2(t) reads the slot of frame t-2
      if (!tap0) x_load(t);
      scale = 0;
      int s2 = 0;
      for (int a = 0; a < 3; ++a) {
        const int tv = t - 2 + a;
        if (tv < 0 && !front) continue;
        const uint32_t hs = (kCache ? slot_of(tv) : h_base + (uint32_t)(tv % kHSlots) * kKc * kTile) + (uint32_t)g * 64u * 128u;
        for (int kc = 0; kc < kKc; ++kc) {
          kstep(false, hs + (uint32_t)kc * kTile, scale);
          scale = 1;
          // the wait of step kKc saw the first tap's steps complete in this warp; the group barrier, in every warp
          if (++s2 == kKc + 1 && tap0) { wg_sync(); x_load(t); }
        }
      }
      finish();
      // ---- E2(t): out = acc + b2 + x; out2 = act(LN_next(out)) from the bf16-rounded out
      mbar_wait(x_bar(g), xphase);
      xphase ^= 1u;
      const uint32_t xslot = slot_of(t - 2);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const long long off = (pos0[r] + (long long)t * frame) * kC;
        const int row = rbase + 8 * r;
        uint8_t* xs = smem_gen + (xslot - smem_base);
        float s = 0.f, q = 0.f;
#pragma unroll
        for (int j = 0; j < kC / 8; ++j) {
          const int c = 8 * j + cq;
          const int cc = c & 63;
          uint32_t* xo = reinterpret_cast<uint32_t*>(xs + (c >> 6) * kTile + swz128_unit(row, cc >> 3) + (cc & 7) * 2);
          const uint32_t xw = *xo;
          const float f0 = acc[4 * j + 2 * r] + bias2[c] + bf16_lo(xw), f1 = acc[4 * j + 2 * r + 1] + bias2[c + 1] + bf16_hi(xw);
          s += f0 + f1;
          q = fmaf(f0, f0, q);
          q = fmaf(f1, f1, q);
          const uint32_t kp = pack_bf16x2(f0, f1);
          *xo = kp;
          acc[4 * j + 2 * r] = bf16_lo(kp);
          acc[4 * j + 2 * r + 1] = bf16_hi(kp);
        }
        if (!p.ln_out) continue;
        const float mean = quad_sum(s) * (1.0f / kC);
        float var = fmaf(-mean, mean, quad_sum(q) * (1.0f / kC));
        var = var < 0.f ? 0.f : var;
        const float rstd = rsqrtf(var + 1e-6f);
        const float nmr = -mean * rstd;
        bf16* o2 = p.out2 + off;
#pragma unroll
        for (int j = 0; j < kC / 8; ++j) {
          const int c = 8 * j + cq;
          float y0 = fmaf(fmaf(acc[4 * j + 2 * r], rstd, nmr), g3[c], b3[c]);
          float y1 = fmaf(fmaf(acc[4 * j + 2 * r + 1], rstd, nmr), g3[c + 1], b3[c + 1]);
          if (p.ln_out_silu) {
            y0 = fmaf(y0, tanh_approx(y0), y0);
            y1 = fmaf(y1, tanh_approx(y1), y1);
          }
          *reinterpret_cast<uint32_t*>(o2 + c) = pack_bf16x2(y0, y1);
        }
      }
      fence_async_smem();
      wg_sync();
      if (gtid == 0) {
        for (int kc = 0; kc < kKc; ++kc)
          tma_store_5d(&maps.out, xslot + (uint32_t)g * 64u * 128u + (uint32_t)kc * kTile, kc * 64, box_w, box_h, t, b);
        bulk_commit();
      }
    }
    if (kCache) {
      // next caches: frames T-2, T-1 of [cache | chunk] (zero padding in front of the first chunk).  The LN2(h) frames are
      // in the ring: the last E1 was followed by a group barrier, and the next write to the ring comes after another.
      for (int j = 0; j < 2; ++j) {
        const int tv = p.T - 2 + j;
        for (int i = gtid; i < 64 * 16; i += 128) {
          int row;
          const long long off = cache_pos(i, j, row);
          const long long pix = off - (((long long)b * 2 + j) * frame) * kC;   // (h, w, c) offset within a frame
          uint4 hv = make_uint4(0u, 0u, 0u, 0u), nv = hv;
          if (tv >= 0 || front) hv = *ring_unit(slot_of(tv), row, (i & 15) * 8);
          if (tv >= 0) nv = *reinterpret_cast<const uint4*>(p.n1 + (((long long)b * p.T + tv) * frame) * kC + pix);
          else if (front) nv = *reinterpret_cast<const uint4*>(p.cn1_in + (((long long)b * 2 + tv + 2) * frame) * kC + pix);
          *reinterpret_cast<uint4*>(p.ch_out + off) = hv;
          *reinterpret_cast<uint4*>(p.cn1_out + off) = nv;
        }
      }
    }
  }
  if (gtid == 0) bulk_wait<0>();   // the last bulk store has read shared memory before the CTA exits
}

// strip box of 128 positions that tiles H x W exactly: the widest power-of-two BW <= 128 dividing W, BH = 128 / BW
bool strip_box(int H, int W, int& BW, int& BH) {
  for (int bw = 128; bw >= 1; bw >>= 1) {
    if (W % bw != 0) continue;
    const int bh = 128 / bw;
    if (bh <= 256 && H % bh == 0) { BW = bw; BH = bh; return true; }
  }
  return false;
}
}  // namespace

const char* tblock_tc_last_error() { return g_tb_err.c_str(); }

bool tblock_tc_supported(int B, int T, int H, int W, int C) {
  g_tb_err.clear();
  if (C != kC) { g_tb_err = "C != 128"; return false; }
  if (B <= 0 || T <= 0) { g_tb_err = "empty"; return false; }
  int BW, BH;
  if (!strip_box(H, W, BW, BH)) { g_tb_err = "H x W not tileable by a 128-position box"; return false; }
  return true;
}

// n1, x, out, out2: dense channels-last bf16 [B,T,H,W,128]; w1, w2: packed [128][3*128] bf16 (k = tap*128 + ci);
// bias*, gamma*, beta*: fp32 [128].  out2 / gamma_out / beta_out may be null (no fused next-stage LayerNorm).
cudaError_t launch_tblock_tc(const bf16* n1, const bf16* x, const bf16* w1, const float* bias1, const float* gamma2,
                             const float* beta2, const bf16* w2, const float* bias2, bf16* out, bf16* out2,
                             const float* gamma_out, const float* beta_out, bool out_silu, int B, int T, int H, int W,
                             cudaStream_t s, const TbCache* cache) {
  g_tb_err.clear();
  if (!tmap_encoder()) { g_tb_err = "cuTensorMapEncodeTiled unavailable"; return cudaErrorNotSupported; }
  TbParams p;
  memset(&p, 0, sizeof(p));
  if (!strip_box(H, W, p.BW, p.BH)) { g_tb_err = "H x W not tileable"; return cudaErrorInvalidValue; }
  p.B = B; p.T = T; p.H = H; p.W = W;
  p.tilesW = W / p.BW; p.tilesH = H / p.BH;
  p.num_strips = (long long)B * p.tilesH * p.tilesW;
  p.bias1 = bias1; p.bias2 = bias2; p.g2 = gamma2; p.b2 = beta2;
  p.ln_out = (out2 && gamma_out && beta_out) ? 1 : 0;
  p.ln_out_silu = out_silu ? 1 : 0;
  p.g3 = gamma_out; p.b3 = beta_out;
  p.x = x; p.out = out; p.out2 = out2;
  if (cache) {
    if (!cache->n1_out || !cache->h_out || (!cache->n1_in != !cache->h_in)) { g_tb_err = "cache: both outputs, and both or no inputs"; return cudaErrorInvalidValue; }
    p.n1 = n1;
    p.cached_in = cache->n1_in ? 1 : 0;
    p.cn1_in = cache->n1_in; p.ch_in = cache->h_in; p.cn1_out = cache->n1_out; p.ch_out = cache->h_out;
  }
  const size_t fixed = 1024 + (size_t)kHSlots * kKc * kTile + 16 + 6 * kC * 4;
  const size_t budget = 225 * 1024;
  int stages = (int)((budget - fixed) / (2 * kTile + 16));
  if (stages > 4) stages = 4;
  p.stages = stages;
  const size_t smem = fixed + (size_t)stages * (2 * kTile + 16);
  TbMaps maps;
  {
    cuuint64_t dims[5] = {(cuuint64_t)kC, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)T, (cuuint64_t)B};
    cuuint64_t strides[4] = {(cuuint64_t)kC * 2, (cuuint64_t)W * kC * 2, (cuuint64_t)H * W * kC * 2, (cuuint64_t)T * H * W * kC * 2};
    cuuint32_t box[5] = {64, (cuuint32_t)p.BW, (cuuint32_t)p.BH, 1, 1};
    if (!encode_tmap_16b(&maps.n1, 5, n1, dims, strides, box, "n1", g_tb_err)) return cudaErrorInvalidValue;
    maps.cn1 = maps.n1;
    // x and out: one consumer warpgroup's 64 rows of a strip, the rows (h, w) in strip order
    const int bw = p.BW < 64 ? p.BW : 64;
    cuuint32_t box64[5] = {64, (cuuint32_t)bw, (cuuint32_t)(64 / bw), 1, 1};
    for (int i = 0; i < 2; ++i)
      if (!encode_tmap_16b(i ? &maps.out : &maps.x, 5, i ? (const void*)out : x, dims, strides, box64, "x / out", g_tb_err))
        return cudaErrorInvalidValue;
    if (p.cached_in) {
      dims[3] = 2;
      strides[3] = 2ull * H * W * kC * 2;
      if (!encode_tmap_16b(&maps.cn1, 5, p.cn1_in, dims, strides, box, "n1 cache", g_tb_err)) return cudaErrorInvalidValue;
    }
  }
  for (int i = 0; i < 2; ++i) {
    cuuint64_t dims[3] = {(cuuint64_t)(3 * kC), (cuuint64_t)kC, 1};
    cuuint64_t strides[2] = {(cuuint64_t)(3 * kC) * 2, (cuuint64_t)(3 * kC) * kC * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)kC, 1};
    if (!encode_tmap_16b(i ? &maps.w2 : &maps.w1, 3, i ? w2 : w1, dims, strides, box, "weights", g_tb_err)) return cudaErrorInvalidValue;
  }
  int dev = 0;
  const cudaError_t dev_err = current_device(dev);
  if (dev_err != cudaSuccess) { g_tb_err = "no current device, or its index is out of range"; return dev_err; }
  {
    static SmemLimitOnce smem_limit;
    const cudaError_t e = smem_limit.ensure(dev, 227 * 1024, tblock_tc_kernel<false>, tblock_tc_kernel<true>);
    if (e != cudaSuccess) { g_tb_err = "cudaFuncSetAttribute(smem)"; return e; }
  }
  const int num_sms = device_sms(dev);
  const unsigned grid = (unsigned)(p.num_strips < num_sms ? p.num_strips : num_sms);
  const double M = (double)B * T * H * W;
  char det[96] = "";
  if (prof_enabled()) snprintf(det, sizeof(det), cache ? "strip %dx%d T%d ln_out%d cache%d" : "strip %dx%d T%d ln_out%d", p.BH, p.BW, T,
                               p.ln_out, p.cached_in);
  ProfScope _ps("tblock_tc", 2.0 * 2.0 * M * 3 * kC * kC, 2.0 * M * kC * (3.0 + (p.ln_out ? 1.0 : 0.0)), s, det);
  if (cache) tblock_tc_kernel<true><<<grid, kThreadsTb, smem, s>>>(maps, p);
  else tblock_tc_kernel<false><<<grid, kThreadsTb, smem, s>>>(maps, p);
  count_launch();
  return cudaGetLastError();
}

}  // namespace vt
