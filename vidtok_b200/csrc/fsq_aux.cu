// FSQ auxiliary loss (regularizers.py:232-245: clamped per-sample entropy, codebook entropy of the batch-mean distribution,
// commitment MSE) without the tokens x codebook distance / softmax matrices the reference materialises.
//
// The implicit codebook is a product grid, so logit_j = 2 inv_T sum_i z_i c_i(k_i(j)) and the softmax over the codebook is a
// product of one small softmax per latent channel: p_j = prod_i q_i(k_i(j)), q_i = softmax_k(2 inv_T z_i c_i(k)).
//  * per-sample entropy with the 1e-5 clamp: since sum_j p_j = 1, H = sum_{p>=eps} -p log p - log(eps) (1 - sum_{p>=eps} p).
//    Only entries with p >= eps are visited: a depth-first walk over the digits that prunes a prefix whose partial product
//    is below eps (every further factor is <= 1).  -p log p = -p sum_i log q_i, so a leaf costs one multiply and one FMA.
//  * avg_prob_j = mean_n p_nj is a sum of rank-1 products: with the digits split into a low and a high group,
//    avg[j_hi][j_lo] = 1/N sum_n Hi_n(j_hi) Lo_n(j_lo), a GEMM over the tokens in fp32 FMA (tf32 would give ~1e-3).  The
//    operand tiles are formed in shared memory from the per-token factor tables, so only N x sum(L) floats are stored.
// Every reduction runs in a fixed order (no atomics): two runs give the same bits.
#include <cmath>

#include "common.cuh"
#include "kernels.h"

namespace vt {
namespace {

constexpr int kWarps = 8, kTokPerWarp = 4, kTokPerBlock = kWarps * kTokPerWarp;
constexpr int kBM = 64, kBN = 64, kBK = 16;
constexpr float kEps = 1e-5f;   // regularizers.py:41-42 (clamp(min=eps) of an fp32 tensor)

size_t align256(size_t n) { return (n + 255) / 256 * 256; }

// workspace: per-token factor tables Q [N][SL] | per-block (entropy, commit) sums [nblk] | per-K-slice avg_prob [ksplit][J]
struct AuxPlan {
  FsqAuxGeom g;
  long long nblk;
  size_t q_bytes, blk_bytes, part_bytes;
};

AuxPlan plan_aux(const FsqAuxGeom& g) {
  AuxPlan p;
  p.g = g;
  p.nblk = (g.N + kTokPerBlock - 1) / kTokPerBlock;
  p.q_bytes = align256((size_t)g.N * g.SL * sizeof(float));
  p.blk_bytes = align256((size_t)p.nblk * sizeof(double2));
  p.part_bytes = align256((size_t)g.ksplit * g.J * sizeof(float));
  return p;
}

// ---- token pass: factor tables, clamped per-sample entropy, squared commit error ----------------------------------------
// One warp per token (kTokPerWarp tokens in turn).  Lanes < d build channel i's softmax table (double, stored fp32); the
// entropy walk splits the first min(2, d-1) digits across the lanes.
__global__ void __launch_bounds__(256) fsq_aux_tokens_kernel(const float* __restrict__ h, FsqAuxGeom g, FsqConst fc, long long P,
                                                             float inv_t, float* __restrict__ Q, double2* __restrict__ blk) {
  __shared__ float tab[kWarps][2][VT_FSQ_AUX_MAX_SUM_LEVELS];
  __shared__ double2 wsum[kWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sq = tab[warp][0];
  float* slq = tab[warp][1];
  const int d = g.d, last = d - 1, mp = d >= 3 ? 2 : d - 1;
  int M = 1;
  for (int i = 0; i < mp; ++i) M *= g.L[i];
  const int Ll = g.L[last], offl = g.off[last];
  double accH = 0.0, accC = 0.0;
  for (int t = 0; t < kTokPerWarp; ++t) {
    const long long n = (long long)blockIdx.x * kTokPerBlock + warp * kTokPerWarp + t;
    if (n >= g.N) break;   // warp-uniform
    const long long b = n / P, pos = n % P;
    double ce = 0.0;
    if (lane < d) {
      const int i = lane, L = g.L[i], hw = L / 2, off = g.off[i];
      const float z = h[(b * d + i) * P + pos];
      float idx_unused = 0.f;
      const double e = (double)z - (double)fsq_code(fc, i, z, idx_unused);
      ce = e * e;
      const double zs = 2.0 * (double)inv_t * (double)z;
      double m = -INFINITY;
      for (int k = 0; k < L; ++k) m = fmax(m, zs * (double)__fdiv_rn((float)(k - hw), (float)hw));
      double s = 0.0;
      for (int k = 0; k < L; ++k) s += exp(zs * (double)__fdiv_rn((float)(k - hw), (float)hw) - m);
      const double ls = log(s);
      for (int k = 0; k < L; ++k) {
        const double lq = zs * (double)__fdiv_rn((float)(k - hw), (float)hw) - m - ls;
        const float q = (float)exp(lq);
        sq[off + k] = q;
        slq[off + k] = (float)lq;
        Q[n * g.SL + off + k] = q;
      }
    }
    __syncwarp();
    double hs = 0.0, ms = 0.0;
    for (int c = lane; c < M; c += 32) {
      float P0 = 1.f, S0 = 0.f;
      int r = c;
      for (int i = 0; i < mp; ++i) {
        const int k = r % g.L[i];
        r /= g.L[i];
        P0 *= sq[g.off[i] + k];
        S0 += slq[g.off[i] + k];
      }
      if (P0 < kEps) continue;
      int kk[VT_MAX_FSQ];
      float Pp[VT_MAX_FSQ], Sp[VT_MAX_FSQ];
      int lv = mp;
      Pp[lv] = P0; Sp[lv] = S0; kk[lv] = 0;
      while (true) {
        if (lv == last) {
          const float Pt = Pp[lv], St = Sp[lv];
          float hl = 0.f, ml = 0.f;
          for (int k = 0; k < Ll; ++k) {
            const float p = Pt * sq[offl + k];
            if (p >= kEps) { hl = fmaf(p, St + slq[offl + k], hl); ml += p; }
          }
          hs += (double)hl;
          ms += (double)ml;
          if (lv == mp) break;
          --lv; ++kk[lv];
          continue;
        }
        if (kk[lv] == g.L[lv]) {
          if (lv == mp) break;
          --lv; ++kk[lv];
          continue;
        }
        const float p = Pp[lv] * sq[g.off[lv] + kk[lv]];
        if (p < kEps) { ++kk[lv]; continue; }
        Pp[lv + 1] = p;
        Sp[lv + 1] = Sp[lv] + slq[g.off[lv] + kk[lv]];
        kk[lv + 1] = 0;
        ++lv;
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      hs += __shfl_xor_sync(0xffffffffu, hs, o);
      ms += __shfl_xor_sync(0xffffffffu, ms, o);
      ce += __shfl_xor_sync(0xffffffffu, ce, o);
    }
    accH += -hs - log((double)kEps) * (1.0 - ms);   // sum_{p>=eps} -p log p - log(eps) * (mass below eps)
    accC += ce;
    __syncwarp();   // the tables are rewritten for the next token
  }
  if (lane == 0) wsum[warp] = make_double2(accH, accC);
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, c = 0.0;
    for (int w = 0; w < kWarps; ++w) { a += wsum[w].x; c += wsum[w].y; }
    blk[blockIdx.x] = make_double2(a, c);
  }
}

// ---- contraction: part[ks][j_hi * Jlo + j_lo] = sum over the tokens of K slice ks of Hi_n(j_hi) * Lo_n(j_lo) --------------
// 64 x 64 output tile per block, 4 x 4 per thread, 16 tokens per step; each step's products are summed on their own before
// they join the running sum (shorter fp32 accumulation chains).
__global__ void __launch_bounds__(256) fsq_aux_avgprob_kernel(const float* __restrict__ Q, FsqAuxGeom g, float* __restrict__ part) {
  __shared__ float Qs[kBK][VT_FSQ_AUX_MAX_SUM_LEVELS];
  __shared__ float As[kBK][kBM], Bs[kBK][kBN];
  __shared__ short hiOff[kBM][VT_MAX_FSQ], loOff[kBN][VT_MAX_FSQ];
  __shared__ bool hiOk[kBM], loOk[kBN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int jh0 = blockIdx.y * kBM, jl0 = blockIdx.x * kBN, ks = blockIdx.z;
  const int nh = g.d - g.a, nl = g.a;
  const long long n0 = (long long)ks * g.kchunk, n1 = min(g.N, n0 + g.kchunk);
  if (tid < kBM) {
    int j = jh0 + tid;
    hiOk[tid] = j < g.Jhi;
    for (int i = 0; i < nh; ++i) { hiOff[tid][i] = (short)(g.off[g.a + i] + j % g.L[g.a + i]); j /= g.L[g.a + i]; }
  } else if (tid < kBM + kBN) {
    const int c = tid - kBM;
    int j = jl0 + c;
    loOk[c] = j < g.Jlo;
    for (int i = 0; i < nl; ++i) { loOff[c][i] = (short)(g.off[i] + j % g.L[i]); j /= g.L[i]; }
  }
  float acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
  for (long long nb = n0; nb < n1; nb += kBK) {
    __syncthreads();
    for (int e = tid; e < kBK * g.SL; e += 256) {
      const int r = e / g.SL, c = e % g.SL;
      Qs[r][c] = nb + r < n1 ? Q[(nb + r) * g.SL + c] : 0.f;
    }
    __syncthreads();
    for (int e = tid; e < kBK * kBM; e += 256) {
      const int r = e / kBM, c = e % kBM;
      float v = 0.f;
      if (hiOk[c]) {
        v = 1.f;
        for (int i = 0; i < nh; ++i) v *= Qs[r][hiOff[c][i]];
      }
      As[r][c] = v;
    }
    for (int e = tid; e < kBK * kBN; e += 256) {
      const int r = e / kBN, c = e % kBN;
      float v = 0.f;
      if (loOk[c]) {   // the low group is never empty, so padding tokens (Q = 0) contribute 0
        v = 1.f;
        for (int i = 0; i < nl; ++i) v *= Qs[r][loOff[c][i]];
      }
      Bs[r][c] = v;
    }
    __syncthreads();
    float stp[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) stp[r][c] = 0.f;
#pragma unroll
    for (int k = 0; k < kBK; ++k) {
      float a[4], bv[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) a[r] = As[k][ty + 16 * r];
#pragma unroll
      for (int c = 0; c < 4; ++c) bv[c] = Bs[k][tx + 16 * c];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) stp[r][c] = fmaf(a[r], bv[c], stp[r][c]);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[r][c] += stp[r][c];
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int jh = jh0 + ty + 16 * r;
    if (jh >= g.Jhi) continue;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int jl = jl0 + tx + 16 * c;
      if (jl < g.Jlo) part[(size_t)ks * g.J + (size_t)jh * g.Jlo + jl] = acc[r][c];
    }
  }
}

// ---- K slices -> avg_prob (mean over the tokens); block 0 also reduces the token pass's per-block sums -------------------
__global__ void __launch_bounds__(256) fsq_aux_reduce_kernel(const float* __restrict__ part, const double2* __restrict__ blk,
                                                             long long nblk, FsqAuxGeom g, float* __restrict__ stats,
                                                             float* __restrict__ avg) {
  const long long j = (long long)blockIdx.x * 256 + threadIdx.x;
  if (j < g.J) {
    double s = 0.0;
    for (int ks = 0; ks < g.ksplit; ++ks) s += (double)part[(size_t)ks * g.J + j];
    avg[j] = (float)(s / (double)g.N);
  }
  if (blockIdx.x != 0) return;
  __shared__ double2 red[256];
  double a = 0.0, c = 0.0;
  for (long long i = threadIdx.x; i < nblk; i += 256) { a += blk[i].x; c += blk[i].y; }
  red[threadIdx.x] = make_double2(a, c);
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      red[threadIdx.x].x += red[threadIdx.x + w].x;
      red[threadIdx.x].y += red[threadIdx.x + w].y;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    stats[0] = (float)(red[0].x / (double)g.N);              // per_sample_entropy
    stats[1] = (float)(red[0].y / ((double)g.N * g.d));      // commit_loss = mean((z - codes)^2)
  }
}

// ---- finish: codebook entropy per segment over the whole codebook, weighted terms, mean over the segments ---------------
__global__ void __launch_bounds__(1024) fsq_aux_finish_kernel(const float* __restrict__ stats, const float* __restrict__ avg,
                                                              int nseg, int J, int world, float w_ent, float gamma, float w_commit,
                                                              float* __restrict__ aux, float* __restrict__ comp) {
  __shared__ double red[32];
  const int tid = threadIdx.x;
  float total = 0.f;
  for (int s = 0; s < nseg; ++s) {
    double e = 0.0;
    for (int j = tid; j < J; j += 1024) {
      float a = avg[(size_t)s * J + j];
      if (world > 1) a = __fdiv_rn(a, (float)world);   // maybe_distributed_mean (regularizers.py:49-59) after the sum
      e -= (double)a * log((double)fmaxf(a, kEps));
    }
    for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
    if ((tid & 31) == 0) red[tid >> 5] = e;
    __syncthreads();
    if (tid < 32) {
      double v = red[tid];
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (tid == 0) {
        // fp32 op by op as regularizers.py:243-245,264-266 evaluates it (no FMA contraction)
        const float pse = stats[2 * s], commit = stats[2 * s + 1], cbe = (float)v;
        const float ent = __fsub_rn(pse, __fmul_rn(gamma, cbe));
        const float a = __fadd_rn(__fmul_rn(ent, w_ent), __fmul_rn(commit, w_commit));
        total = __fadd_rn(total, a);
        if (comp) {
          comp[4 * s + 0] = pse;
          comp[4 * s + 1] = cbe;
          comp[4 * s + 2] = commit;
          comp[4 * s + 3] = a;
        }
      }
    }
    __syncthreads();
  }
  if (tid == 0) *aux = __fdiv_rn(total, (float)nseg);   // tile_encode: torch.mean over the chunks (autoencoder_v1_1.py:261-264)
}

}  // namespace

const char* fsq_aux_geometry(int d, const int* levels, long long N, FsqAuxGeom* g) {
  if (d < 1 || d > VT_MAX_FSQ) return "FSQ aux loss: 1 <= len(levels) <= 8 required";
  if (N <= 0) return "FSQ aux loss: no tokens";
  *g = FsqAuxGeom();
  g->d = d;
  g->N = N;
  long long J = 1;
  int sl = 0;
  for (int i = 0; i < d; ++i) {
    if (levels[i] < 2) return "FSQ aux loss: every level must be >= 2 (a level of 1 has no code spacing)";
    g->L[i] = levels[i];
    g->off[i] = sl;
    sl += levels[i];
    J *= levels[i];
    if (J > VT_FSQ_AUX_MAX_CODEBOOK) return "FSQ aux loss: codebook larger than 2^22 codes";
  }
  if (sl > VT_FSQ_AUX_MAX_SUM_LEVELS) return "FSQ aux loss: sum of the levels larger than 256";
  g->SL = sl;
  g->J = (int)J;
  // low digit group: the split whose two factor counts are closest (ties: the larger low group); never empty
  long long lo = 1, best = -1;
  for (int a = 1; a <= d; ++a) {
    lo *= levels[a - 1];
    const long long hi = J / lo;
    const long long diff = lo > hi ? lo - hi : hi - lo;
    if (best < 0 || diff <= best) { best = diff; g->a = a; g->Jlo = (int)lo; g->Jhi = (int)hi; }
  }
  const long long tiles = (long long)((g->Jlo + kBN - 1) / kBN) * ((g->Jhi + kBM - 1) / kBM);
  long long ks = std::max(1LL, 256 / tiles);
  ks = std::min(ks, std::max(1LL, (1LL << 20) / J));          // K-slice partials stay within 4 MB
  ks = std::min(ks, (N + kBK - 1) / kBK);
  g->ksplit = (int)ks;
  g->kchunk = ((N + ks - 1) / ks + kBK - 1) / kBK * kBK;
  return nullptr;
}

size_t fsq_aux_workspace(const FsqAuxGeom& g) {
  const AuxPlan p = plan_aux(g);
  return p.q_bytes + p.blk_bytes + p.part_bytes;
}

cudaError_t launch_fsq_aux_partials(const float* h, const FsqAuxGeom& g, const int* levels, long long P, float inv_t, float* stats,
                                    float* avg_prob, void* ws, cudaStream_t s) {
  const AuxPlan p = plan_aux(g);
  char* w = (char*)ws;
  float* Q = (float*)w;
  double2* blk = (double2*)(w + p.q_bytes);
  float* part = (float*)(w + p.q_bytes + p.blk_bytes);
  const FsqConst fc = make_fsq_const(g.d, levels);
  {
    ProfScope _ps("fsq_aux_tokens", (double)g.N * g.SL * 8.0, (double)g.N * (g.d + g.SL) * 4.0, s);
    fsq_aux_tokens_kernel<<<(unsigned)p.nblk, 256, 0, s>>>(h, g, fc, P, inv_t, Q, blk);
    count_launch();
  }
  {
    const dim3 grid((g.Jlo + kBN - 1) / kBN, (g.Jhi + kBM - 1) / kBM, g.ksplit);
    ProfScope _ps("fsq_aux_avgprob", 2.0 * (double)g.N * g.J,
                  (double)g.N * g.SL * 4.0 * grid.x * grid.y + (double)g.ksplit * g.J * 4.0, s);
    fsq_aux_avgprob_kernel<<<grid, 256, 0, s>>>(Q, g, part);
    count_launch();
  }
  {
    ProfScope _ps("fsq_aux_reduce", (double)g.ksplit * g.J, ((double)g.ksplit + 1.0) * g.J * 4.0 + (double)p.nblk * 16.0, s);
    fsq_aux_reduce_kernel<<<(unsigned)((g.J + 255) / 256), 256, 0, s>>>(part, blk, p.nblk, g, stats, avg_prob);
    count_launch();
  }
  return cudaGetLastError();
}

cudaError_t launch_fsq_aux_finalize(const float* stats, const float* avg_prob, int nseg, int J, int world, float w_ent, float gamma,
                                    float w_commit, float* aux, float* comp, cudaStream_t s) {
  ProfScope _ps("fsq_aux_finish", 3.0 * (double)nseg * J, (double)nseg * (J + 2) * 4.0, s);
  fsq_aux_finish_kernel<<<1, 1024, 0, s>>>(stats, avg_prob, nseg, J, world, w_ent, gamma, w_commit, aux, comp);
  count_launch();
  return cudaGetLastError();
}

}  // namespace vt
