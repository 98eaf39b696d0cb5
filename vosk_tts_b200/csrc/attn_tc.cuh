// attn_tc.cuh -- windowed relative-position multi-head self-attention (attentions.py:165-196) on the Hopper tensor cores
// (wgmma + TMA + mbarrier), sm_90a.  One CTA = 128 query rows of one head of one utterance.
//
//   S  = Q K^T            128 x 64 key tile, fp32 in registers                  (attentions.py:172, scores)
//   Sr = Q Ek^T           128 x 16 (9 relative offsets, zero padded), once      (:173-177, rel_logits before the skew)
//   s_ij = (S_ij + [|j-i|<=W] Sr_i[j-i+W]) / sqrt(dk);  keys >= len masked      (:178,183: -1e4 fill == exp -> 0 in fp32)
//   P  = exp(s - m)       online softmax, running max refreshed lazily          (:190 softmax)
//   O += P V + Pband Ev   128 x dk, fp32 in registers                           (:192-196, output + relative values)
//   out = O / l
//
// Operand format = the split-bf16 planes of the tensor-core convs: x = hi + lo to ~2^-18, three MMAs per K16 slice
// (lo*hi + hi*lo + hi*hi).  Q, K: K-major 128B-swizzled TMA tiles of the qkv planes (channels-last, so a head is a
// channel range and no transposition is needed).  V is consumed as an MN-major B operand straight from the same
// channels-last tiles.  P never leaves the registers: the S accumulator fragment of a K16 slice of keys is exactly the
// A-operand fragment of the P V MMA, so P is split into bf16 hi/lo pairs in place.  The relative-position terms ride on
// the same tensor-core path: Q Ek^T is one extra N=16 MMA group per CTA, and P_band Ev one extra K=16 MMA per diagonal
// key tile (its A fragment is gathered from a small per-row band scratch in shared memory).
//
// Warp roles (288 threads): warps 0..7 = two consumer warpgroups of 64 query rows each (MMAs, softmax with the row
// statistics reduced over the 4 lanes that share a row, O rescaling and the epilogue); warp 8 = TMA producer.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "wgmma.cuh"

namespace vtts {

constexpr int ATC_BM = 128;        // query rows per CTA
constexpr int ATC_KT = 64;         // keys per tile
constexpr int ATC_NS = 2;          // K/V ring depth
constexpr int ATC_CWG = 2;         // consumer warpgroups
constexpr int ATC_THREADS = ATC_CWG * 128 + 32;
constexpr int ATC_RELP = 16;       // relative-offset slots (2W+1 <= 16)
constexpr int ATC_RS = 13;         // floats per row of the per-row band scratch in shared memory
constexpr float ATC_LAZY = 6.0f;   // the running max is refreshed only when a tile exceeds it by more than this (natural log units)

struct AttnTcParams {
  CUtensorMap q_hi, q_lo;      // qkv planes [rows][ld], box 64 channels x 128 rows
  CUtensorMap kv_hi, kv_lo;    // same planes, box 64 channels x 64 rows
  CUtensorMap rk_hi, rk_lo;    // relative-key table   [16][128] bf16 (rows >= 2W+1 and channels >= dk are zero), box 64 x 16
  CUtensorMap rv_hi, rv_lo;    // relative-value table [16][128]
  float* out;                  // fp32 rows [.][ldo] (or null)
  __nv_bfloat16* p_hi;         // split-bf16 planes of the output for a tensor-core consumer (or null)
  __nv_bfloat16* p_lo;
  int ldo, ldp;
  int n_heads, window;
  int koff, voff;              // channel offsets of the K and V sections inside a qkv row (H, 2H)
};

constexpr int atc_chunks(int dk) { return (dk + 63) / 64; }
constexpr int atc_smem_bytes(int dk) {
  return 2 * atc_chunks(dk) * ATC_BM * 128                 // Q hi/lo
         + ATC_NS * 2 * 2 * atc_chunks(dk) * ATC_KT * 128  // K and V hi/lo per stage
         + 2 * 2 * atc_chunks(dk) * ATC_RELP * 128         // relative key / value tables hi/lo
         + 2 * ATC_BM * ATC_RS * 4                         // per-row band scratch (Sr values, band P values)
         + 1024 /*alignment slack*/ + 256 /*barriers*/;
}

__device__ __forceinline__ float lds_f32(uint32_t saddr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(saddr));
  return v;
}
__device__ __forceinline__ void sts_f32(uint32_t saddr, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(saddr), "f"(v) : "memory"); }

template <int N>
__device__ __forceinline__ void atc_pv(float* d, const uint32_t (&a)[4], uint64_t db) {
  if constexpr (N == 64) wgmma_rs_n64(d, a, db);
  else wgmma_rs_n32(d, a, db);
}

template <int DK>
__global__ void __launch_bounds__(ATC_THREADS, 1)
attn_tc_kernel(const __grid_constant__ AttnTcParams ap, const int* __restrict__ lens, const int* __restrict__ offs) {
  static_assert(DK % 32 == 0 && DK >= 32 && DK <= 128, "head dim must be 32/64/96/128");
  constexpr int NC = atc_chunks(DK);                 // 64-channel chunks of a head (the last one may be half used)
  constexpr int LASTW = DK - 64 * (NC - 1);          // channels used of the last chunk
  constexpr int Q_TILE = ATC_BM * 128, KV_TILE = ATC_KT * 128, R_TILE = ATC_RELP * 128;
  constexpr int STAGE_BYTES = 2 * 2 * NC * KV_TILE;  // K hi/lo + V hi/lo
  PDL_LAUNCH();
  const int b = blockIdx.z, head = blockIdx.y;
  const int q0 = blockIdx.x * ATC_BM;
  // lens/offs are final before the graph that contains this kernel starts (host copies or the previous phase): an idle
  // CTA leaves before it initialises anything
  const int len = lens[b];
  if (q0 >= len) return;
  const long base = offs[b];
  const int W = ap.window, nrel = 2 * W + 1;

  extern __shared__ uint8_t atc_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(atc_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sQ = smem;                                   // [plane][chunk][128 x 128 B]
  uint8_t* sKV = sQ + 2 * NC * Q_TILE;                  // [stage][K: plane, chunk | V: plane, chunk][64 x 128 B]
  uint8_t* sRK = sKV + ATC_NS * STAGE_BYTES;            // [plane][chunk][16 x 128 B]
  uint8_t* sRV = sRK + 2 * NC * R_TILE;
  float* sSr = reinterpret_cast<float*>(sRV + 2 * NC * R_TILE);   // [128][RS]  q_i . Ek[m]
  float* sPb = sSr + ATC_BM * ATC_RS;                             // [128][RS]  band probabilities of the current tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(sPb + ATC_BM * ATC_RS);
  uint64_t* q_full = bars;              // Q tile + relative tables landed
  uint64_t* kv_full = bars + 1;         // [NS]
  uint64_t* kv_empty = kv_full + ATC_NS;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nt = (len + ATC_KT - 1) / ATC_KT;

  if (warp == ATC_CWG * 4 && lane == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < ATC_NS; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], ATC_CWG); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&ap.q_hi)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&ap.q_lo)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&ap.kv_hi)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&ap.kv_lo)) : "memory");
  }
  __syncthreads();

  if (warp == ATC_CWG * 4) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      // the relative-position tables are constants: requested before the dependency wait
      mbar_expect_tx(q_full, (uint32_t)(2 * NC * Q_TILE + 4 * NC * R_TILE));
      for (int c = 0; c < NC; ++c) {
        tma_load_2d(sRK + c * R_TILE, &ap.rk_hi, c * 64, 0, q_full);
        tma_load_2d(sRK + (NC + c) * R_TILE, &ap.rk_lo, c * 64, 0, q_full);
        tma_load_2d(sRV + c * R_TILE, &ap.rv_hi, c * 64, 0, q_full);
        tma_load_2d(sRV + (NC + c) * R_TILE, &ap.rv_lo, c * 64, 0, q_full);
      }
      PDL_WAIT();
      timeline_stamp_t(-31);
      const int qch = head * DK;
      for (int c = 0; c < NC; ++c) {
        tma_load_2d(sQ + c * Q_TILE, &ap.q_hi, qch + c * 64, (int)base + q0, q_full);
        tma_load_2d(sQ + (NC + c) * Q_TILE, &ap.q_lo, qch + c * 64, (int)base + q0, q_full);
      }
      for (int t = 0; t < nt; ++t) {
        const int st = t % ATC_NS;
        if (t >= ATC_NS) mbar_wait(&kv_empty[st], ((t / ATC_NS) - 1) & 1);
        uint8_t* kb = sKV + st * STAGE_BYTES;
        uint8_t* vb = kb + 2 * NC * KV_TILE;
        mbar_expect_tx(&kv_full[st], (uint32_t)STAGE_BYTES);
        const int row = (int)base + t * ATC_KT;
        for (int c = 0; c < NC; ++c) {
          tma_load_2d(kb + c * KV_TILE, &ap.kv_hi, ap.koff + qch + c * 64, row, &kv_full[st]);
          tma_load_2d(kb + (NC + c) * KV_TILE, &ap.kv_lo, ap.koff + qch + c * 64, row, &kv_full[st]);
        }
        for (int c = 0; c < NC; ++c) {
          tma_load_2d(vb + c * KV_TILE, &ap.kv_hi, ap.voff + qch + c * 64, row, &kv_full[st]);
          tma_load_2d(vb + (NC + c) * KV_TILE, &ap.kv_lo, ap.voff + qch + c * 64, row, &kv_full[st]);
        }
      }
    }
    return;
  }
  // -------------------------------------------------------------------- consumers: 64 query rows per warpgroup
  const int wg = warp >> 2;
  const int g = lane >> 2, q4 = lane & 3;
  const int wrow0 = wg * 64 + (warp & 3) * 16;             // first tile row of this warp
  int row[2], qi[2];
  uint32_t mySr[2], myPb[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    row[h] = wrow0 + g + 8 * h;
    qi[h] = q0 + row[h];
    mySr[h] = smem_u32(sSr + row[h] * ATC_RS);              // (explicit shared-space accesses: generic LD/ST otherwise)
    myPb[h] = smem_u32(sPb + row[h] * ATC_RS);
  }
  const bool leader = (threadIdx.x & 127) == 0;
  const float scale = 1.0f / sqrtf((float)DK);
  const float L2E = 1.4426950408889634f;
  const uint32_t qoff = (uint32_t)(wg * 64 * 128);         // this warpgroup's 64 rows of the Q tile
  PDL_WAIT();
  mbar_wait(q_full, 0);
  timeline_stamp_t(-32);
  {   // Sr = Q Ek^T (N = 16) -> relative-key logits of this thread's rows in shared memory (indexed by a run-time offset below)
    float sr[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) sr[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const uint64_t qh = gmma_desc_sw128(smem_u32(sQ + c * Q_TILE) + qoff), ql = gmma_desc_sw128(smem_u32(sQ + (NC + c) * Q_TILE) + qoff);
      const uint64_t eh = gmma_desc_sw128(smem_u32(sRK + c * R_TILE)), el = gmma_desc_sw128(smem_u32(sRK + (NC + c) * R_TILE));
      const int nk = (c == NC - 1 ? LASTW : 64) / 16;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        if (kk < nk) {
          const uint64_t adv = (uint64_t)((kk * 32) >> 4);
          wgmma_ss_n16(sr, ql + adv, eh + adv);
          wgmma_ss_n16(sr, qh + adv, el + adv);
          wgmma_ss_n16(sr, qh + adv, eh + adv);
        }
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_touch<8>(sr);
#pragma unroll
    for (int jn = 0; jn < 2; ++jn)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int m = jn * 8 + 2 * q4 + e;
          if (m < ATC_RS) sts_f32(mySr[h] + 4 * m, sr[4 * jn + 2 * h + e] * scale);
        }
    __syncwarp();
  }
  float o[NC][32];
#pragma unroll
  for (int c = 0; c < NC; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // l_run: this thread's share of the row sum
  for (int t = 0; t < nt; ++t) {
    const int st = t % ATC_NS;
    const int k0 = t * ATC_KT;
    mbar_wait(&kv_full[st], (t / ATC_NS) & 1);
    if (threadIdx.x == 0) timeline_stamp_t(-40 - t);
    const uint32_t kb = smem_u32(sKV + st * STAGE_BYTES);
    float s[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const uint64_t qh = gmma_desc_sw128(smem_u32(sQ + c * Q_TILE) + qoff), ql = gmma_desc_sw128(smem_u32(sQ + (NC + c) * Q_TILE) + qoff);
      const uint64_t kh = gmma_desc_sw128(kb + c * KV_TILE), kl = gmma_desc_sw128(kb + (NC + c) * KV_TILE);
      const int nk = (c == NC - 1 ? LASTW : 64) / 16;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        if (kk < nk) {
          const uint64_t adv = (uint64_t)((kk * 32) >> 4);
          wgmma_ss_n64(s, ql + adv, kh + adv);
          wgmma_ss_n64(s, qh + adv, kl + adv);
          wgmma_ss_n64(s, qh + adv, kh + adv);
        }
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_touch<32>(s);
    // does the +-W band of any row of this warpgroup cross the key tile?  (warpgroup-uniform: the band MMA is collective)
    const int g_lo = q0 + wg * 64, g_hi = g_lo + 63;
    const bool band = (k0 + ATC_KT - 1 + W >= g_lo) && (k0 - W <= g_hi);
    const int kvalid = len - k0;                   // columns >= kvalid are beyond the utterance
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int jn = 0; jn < 8; ++jn)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = jn * 8 + 2 * q4 + e;
          float v = s[4 * jn + 2 * h + e] * scale;
          if (band) {
            const int m = c + k0 - qi[h] + W;      // relative slot of key column c
            if ((unsigned)m < (unsigned)nrel) v += lds_f32(mySr[h] + 4 * m);
          }
          if (c >= kvalid) v = -INFINITY;
          s[4 * jn + 2 * h + e] = v;
          mx[h] = fmaxf(mx[h], v);
        }
    float mneg[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      // lazily refreshed running max: O and l are rescaled only when the tile max exceeds it by more than ATC_LAZY
      if (t == 0) {
        m_run[h] = mx[h];
      } else if (mx[h] > m_run[h] + ATC_LAZY) {
        const float alpha = exp2f((m_run[h] - mx[h]) * L2E);
        m_run[h] = mx[h];
        l_run[h] *= alpha;
#pragma unroll
        for (int c = 0; c < NC; ++c)
#pragma unroll
          for (int jn = 0; jn < 8; ++jn) { o[c][4 * jn + 2 * h] *= alpha; o[c][4 * jn + 2 * h + 1] *= alpha; }
      }
      mneg[h] = -m_run[h] * L2E;
    }
    if (band) {
      __syncwarp();                                 // the previous tile's band fragment has been read
#pragma unroll
      for (int h = 0; h < 2; ++h)
        for (int m = q4; m < ATC_RS; m += 4) sts_f32(myPb[h] + 4 * m, 0.f);
      __syncwarp();
    }
#pragma unroll
    for (int jn = 0; jn < 8; ++jn)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float p = exp2f(fmaf(s[4 * jn + 2 * h + e], L2E, mneg[h]));
          l_run[h] += p;
          s[4 * jn + 2 * h + e] = p;
          if (band) {
            const int m = jn * 8 + 2 * q4 + e + k0 - qi[h] + W;
            if ((unsigned)m < (unsigned)nrel) sts_f32(myPb[h] + 4 * m, p);
          }
        }
    // P as the A operand of the P V MMAs: the S fragment of keys [16 kk, 16 kk + 16) is the A fragment of K16 slice kk
    uint32_t ph[4][4], pl[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) split_bf16_pair(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1], ph[kk][r], pl[kk][r]);
    uint32_t bh[4], bl[4];
    if (band) {
      __syncwarp();
      float pv[4][2];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int m = 2 * q4 + e + ((r & 2) ? 8 : 0);
          pv[r][e] = m < ATC_RS ? lds_f32(myPb[r & 1] + 4 * m) : 0.f;
        }
#pragma unroll
      for (int r = 0; r < 4; ++r) split_bf16_pair(pv[r][0], pv[r][1], bh[r], bl[r]);
    }
    const uint32_t vb = kb + 2 * NC * KV_TILE;
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      constexpr int NL = LASTW;
      const uint64_t vh = gmma_desc_sw128(vb + c * KV_TILE), vl = gmma_desc_sw128(vb + (NC + c) * KV_TILE);
      auto pv_mma = [&](const uint32_t (&a)[4], uint64_t db) {
        if (c == NC - 1) atc_pv<NL>(o[c], a, db);
        else atc_pv<64>(o[c], a, db);
      };
#pragma unroll
      for (int kk = 0; kk < ATC_KT / 16; ++kk) {
        const uint64_t adv = (uint64_t)((kk * 16 * 128) >> 4);      // 16 keys = 16 rows of 128 bytes
        pv_mma(pl[kk], vh + adv);
        pv_mma(ph[kk], vl + adv);
        pv_mma(ph[kk], vh + adv);
      }
      if (band) {      // + P_band Ev (K = 16 relative offsets)
        const uint64_t eh = gmma_desc_sw128(smem_u32(sRV + c * R_TILE)), el = gmma_desc_sw128(smem_u32(sRV + (NC + c) * R_TILE));
        pv_mma(bl, eh);
        pv_mma(bh, el);
        pv_mma(bh, eh);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < NC; ++c) wgmma_touch<32>(o[c]);
    if (leader) mbar_arrive(&kv_empty[st]);
    if (threadIdx.x == 0) timeline_stamp_t(-60 - t);
  }
  // ---- epilogue: O / l -> fp32 rows and/or split-bf16 planes
  if (threadIdx.x == 0) timeline_stamp_t(-36);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.f / l;
    if (qi[h] >= len) continue;
    const long orow = base + qi[h];
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int jn = 0; jn < 8; ++jn) {
        if (c == NC - 1 && jn * 8 >= LASTW) continue;
        const int ch = head * DK + c * 64 + jn * 8 + 2 * q4;
        const float v0 = o[c][4 * jn + 2 * h] * inv, v1 = o[c][4 * jn + 2 * h + 1] * inv;
        if (ap.out) *reinterpret_cast<float2*>(ap.out + orow * (long)ap.ldo + ch) = make_float2(v0, v1);
        if (ap.p_hi) {
          uint32_t hi, lo;
          split_bf16_pair(v0, v1, hi, lo);
          *reinterpret_cast<uint32_t*>(ap.p_hi + orow * (long)ap.ldp + ch) = hi;
          *reinterpret_cast<uint32_t*>(ap.p_lo + orow * (long)ap.ldp + ch) = lo;
        }
      }
  }
}

}  // namespace vtts
