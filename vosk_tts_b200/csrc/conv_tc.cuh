// conv_tc.cuh -- dense conv1d-as-GEMM on the Hopper tensor cores (wgmma + TMA + mbarrier rings), sm_90a.
//
//   D[t, co] (fp32, registers) = sum_{tap j} sum_{ci} A_j[t, ci] * W_j[co, ci]
//     A_j = rows (t0 + j*dil - pad .. +128) x 64 channels of the producer's *split-bf16 planes* (hi + lo = fp32
//           value to ~2^-17), K-major, fetched by TMA with the 128-byte swizzle straight from the channels-last
//           activation buffer (im2col-free: a tap shift is just a different TMA row coordinate; rows outside the
//           utterance are zero through TMA out-of-bounds fill or the zeroed gap rows between packed utterances),
//     W_j = 64..128 output channels x 64 input channels of the packed bf16 hi/lo weights of tap j.
//   Three bf16 MMAs per K16 slice (hi*hi + lo*hi + hi*lo, fp32 accumulate) give fp32-class accuracy (~1e-5 rel)
//   at 1/3 of the bf16 tensor rate -- several times the FFMA pipe -- which keeps the waveform inside the 1e-3 budget
//   where single-pass bf16 (4.9e-3) or TF32 (6e-4 at 0.2 amplitude) do not (SURVEY.md section 7 "Hard parts").
//
// Warp roles (288 threads): warps 0..7 = two consumer warpgroups, each issuing wgmma for 64 of the tile's 128 rows with
// the accumulator in registers and then running the epilogue on it (bias/cond/activation/residual -> fp32 rows and/or
// split-bf16 planes for the next conv); warp 8 = TMA producer.  Multi-stage mbarrier rings decouple TMA from the tensor pipe.
#pragma once
#include <type_traits>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "wgmma.cuh"

namespace vtts {

constexpr int TC_BM = 128;        // time rows per CTA (two warpgroups of 64)
constexpr int TC_BK = 64;         // input channels per stage (one 128-byte swizzle atom of bf16)
// ring depths per weight-tile width (BN): the 64-wide kernel has room for deeper rings than the 128-wide one
#ifndef VTTS_TC_AST64
#define VTTS_TC_AST64 3
#endif
#ifndef VTTS_TC_WST64
#define VTTS_TC_WST64 4
#endif
#ifndef VTTS_TC_AST128
#define VTTS_TC_AST128 3
#endif
#ifndef VTTS_TC_WST128
#define VTTS_TC_WST128 4
#endif
template <int BN> constexpr int tc_ast() { return BN == 64 ? VTTS_TC_AST64 : VTTS_TC_AST128; }   // activation-tile ring depth
template <int BN> constexpr int tc_wst() { return BN == 64 ? VTTS_TC_WST64 : VTTS_TC_WST128; }   // weight-tile ring depth
constexpr int TC_CWG = 2;                      // consumer warpgroups
constexpr int TC_THREADS = TC_CWG * 128 + 32;  // + the producer warp
constexpr int TC_MAXP = 4;

enum : int { TCE_RELU = 1, TCE_GATE = 2 };

// One conv of a grouped launch.  TcProblemBase is what the default kernels take as a parameter; TcProblem adds the tensor maps of
// the third operand plane (exact 3-way split).  The launch descriptor is a __grid_constant__ kernel parameter: two more
// 128-byte maps per problem are 1 KB more parameters on every launch of the 68-launch single-utterance chain.
struct TcProblemBase {
  CUtensorMap a_hi, a_lo, w_hi, w_lo;
  __nv_bfloat16* p_mid;       // third output plane (or null)
  const float* bias;
  const float* cond;          // per-utterance vector added before the activation (or null)
  const float* res;           // fp32 residual added to the fp32 output (or null)
  float* y;                   // fp32 output rows (or null)
  __nv_bfloat16* p_hi;        // split-bf16 planes of lrelu(out, pl_slope) for the next conv (or null)
  __nv_bfloat16* p_lo;
  int cond_ld, ldr, roff, ldy, yoff, ldp, poff;
  int Cin, Cout, k, dil, pad;
  int out_mul, out_add;       // output row = t*out_mul + out_add (polyphase ConvTranspose1d)
  int in_extra, out_seq_extra;
  int epi;
  float alpha, pl_slope;
  int split;                  // split-K of this problem's tiles (divides TcBatchScalars::split, the cluster size)
  int cl0;                    // mixed-split launches: index of the problem's first cluster
};
struct TcProblem : TcProblemBase {
  CUtensorMap a_mid, w_mid;   // third planes of the exact 3-way split (np == 3)
};

struct TcBatchScalars {
  int n;
  int rmul;
  int tall;     // 1: one activation tile of 128 + (k-1)*dil rows per channel chunk, taps address it through row-shifted
                //    wgmma descriptors; 0: a fresh 128-row tile per (chunk, tap)
  int a_bytes;  // bytes of one activation plane tile in shared memory (multiple of 1024)
  int baseoff;  // experiment: fill the descriptor base-offset field for row-shifted tiles
  int cn;       // CTAs of a cluster along the channel-tile axis that share (TMA-multicast) one activation tile; 1 = off
  int wpre;     // 1: request the first ring of weight tiles before the dependency wait (latency-bound single-wave launches)
  int np;       // operand planes: 2 = (hi, lo), three MMAs per K16 slice (lo*hi + hi*lo + hi*hi, ~2^-17 relative);
                //   3 = (hi, mid, lo), six MMAs (hl + lh + mm + mh + hm + hh): products exact to the last fp32 bit
  int ast, wst; // ring depths (activation / weight tiles) for this launch
  int dbgskip;  // tuning experiments (timing only, wrong results): 1 = no epilogue stores, 2 = no MMAs issued, 4 = no residual loads
  int wmc;      // persistent launches: 2 = CTA pairs (cluster (2,1,1)) walk adjacent row tiles and share every weight tile: each CTA
                //   fetches half of it and TMA-multicasts it into both (halves the L2 reads of the dominant operand); 1 = off
  int persist;  // 1: 1-D grid of resident CTAs walking the (gx, gy, gz) tile space (machine-filling launches)
  int gx, gy, gz;
  int split;    // cluster split-K: `split` CTAs (cluster dims (1,1,split)) each run a contiguous range of the k-steps of one
                //    output tile, exchange partial accumulators through distributed shared memory and each finish
                //    BN/split of the tile's columns (reduce-scatter; fixed summation order => deterministic).  1 = off
  int mixed;    // 1: the problems' splits differ (TcProblemBase::split).  Grid (1, 1, clusters * split), the clusters of one
                //    problem after another; a cluster of problem p covers split / p.split consecutive output tiles (row tile
                //    fastest, then channel tile, then utterance), each reduced over p.split adjacent ranks
  int nb;       // utterances of the launch
  unsigned long long* dbg;   // optional: %globaltimer stamps of CTA (0,0,0) for tuning (tools/microbench.py)
};
template <class PT, int MP = TC_MAXP>
struct TcBatchT : TcBatchScalars {
  PT p[MP];
};
using TcBatch = TcBatchT<TcProblem>;          // what the host fills
// Parameter of the two-plane kernels: no third-plane maps (3.7 KB -> 2.65 KB of kernel parameters per launch).
template <int MP>
inline TcBatchT<TcProblemBase, MP> tc_lite(const TcBatch& tb) {
  TcBatchT<TcProblemBase, MP> l;
  static_cast<TcBatchScalars&>(l) = tb;
  for (int i = 0; i < MP; ++i) l.p[i] = tb.p[i];               // (slices the third-plane maps off)
  return l;
}
__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
#define TC_STAMP(i) do { if (tb.dbg && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) tb.dbg[i] = gtimer(); } while (0)

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// TMA load whose box lands at the same shared-memory offset in every CTA of `mask` and signals each one's mbarrier
__device__ __forceinline__ void tma_load_2d_mc(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}
__device__ __forceinline__ uint32_t cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// arrive on the mbarrier at this offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t rank) {
  uint32_t ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(smem_u32(bar)), "r"(rank));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(ra) : "memory");
}
// a ring slot shared by `n` CTAs of the cluster (multicast) is released in every one of them
__device__ __forceinline__ void tc_release(uint64_t* bar, int n) {
  if (n > 1) {
    for (int r = 0; r < n; ++r) mbar_arrive_remote(bar, (uint32_t)r);
  } else {
    mbar_arrive(bar);
  }
}

// ---- epilogue: acc (+ split partials) + bias (+ cond) -> gate / ReLU -> x alpha -> + residual -> fp32 rows and/or the
// split-bf16 planes of lrelu(., pl_slope) for the next conv.  A consumer thread finishes its tile share one column pair at a
// time, in both of its rows: every global load of a column pair (bias, cond, the residual of both rows) is issued before any
// of its stores, and the next column pair's loads before the current one's stores.  (y and res may alias -- the in-place
// residuals of the WN stacks and the flow's post conv -- so the compiler keeps loads and stores in source order: one
// (row, column pair) at a time made every pair a serial global round trip.)  Loading later pairs ahead of earlier pairs'
// stores is safe under that aliasing: each element is read and written by the one thread that finishes it, and read first.

// The epilogue operands of one problem, read out of the launch descriptor once per tile.
struct TcEpi {
  const float* bias;
  const float* cond;          // this utterance's conditioning row (or null)
  const float* res;           // (null with dbgskip & 4)
  float* y;
  __nv_bfloat16 *p_hi, *p_lo, *p_mid;
  int ldr, roff, ldy, yoff, ldp, poff;
  int ncol;                   // output channels: Cout, or Cout / 2 behind the gate
  float alpha, pl_slope;
  bool gate, relu, store;     // store: false with dbgskip & 1
};
template <class PT>
__device__ __forceinline__ TcEpi tc_epi(const PT& P, int b, int dbgskip) {
  TcEpi E;
  E.bias = P.bias;
  E.cond = P.cond ? P.cond + (long)b * P.cond_ld : nullptr;
  E.res = (dbgskip & 4) ? nullptr : P.res;
  E.y = P.y;
  E.p_hi = P.p_hi; E.p_lo = P.p_lo; E.p_mid = P.p_mid;
  E.ldr = P.ldr; E.roff = P.roff; E.ldy = P.ldy; E.yoff = P.yoff; E.ldp = P.ldp; E.poff = P.poff;
  E.gate = (P.epi & TCE_GATE) != 0;
  E.relu = (P.epi & TCE_RELU) != 0;
  E.ncol = E.gate ? P.Cout >> 1 : P.Cout;
  E.alpha = P.alpha; E.pl_slope = P.pl_slope;
  E.store = !(dbgskip & 1);
  return E;
}
// One column pair of a consumer thread: accumulator columns (c, c + 1), in each of the thread's two rows.  Gate: the pair
// makes output channel oc = c / 2.
struct TcEpiCol {
  int c, oc, nout;
  bool ok;                    // the pair exists in this thread's share of the tile and has an output channel
};
__device__ __forceinline__ TcEpiCol tc_epi_col(const TcEpi& E, int c, bool in_tile) {
  TcEpiCol k;
  k.c = c;
  k.oc = E.gate ? c >> 1 : c;
  k.ok = in_tile && k.oc < E.ncol;
  k.nout = E.gate ? 1 : min(2, E.ncol - k.oc);
  return k;
}
// The global loads of one column pair: bias and cond of its columns, the residual of each row (rowok: the row lies in the
// utterance).
struct TcEpiIn {
  float b0, b1, c0, c1, r[2][2];
};
__device__ __forceinline__ TcEpiIn tc_epi_load(const TcEpi& E, const TcEpiCol& k, const long (&orow)[2], const bool (&rowok)[2]) {
  TcEpiIn in = {};
  if (!(k.ok && (rowok[0] || rowok[1]))) return in;
  const bool two = E.gate || k.nout > 1;       // columns c and c + 1 are both used
  in.b0 = E.bias[k.c];
  if (two) in.b1 = E.bias[k.c + 1];
  if (E.cond) {
    in.c0 = E.cond[k.c];
    if (two) in.c1 = E.cond[k.c + 1];
  }
  if (E.res) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!rowok[h]) continue;
      const float* rp = E.res + orow[h] * (long)E.ldr + E.roff + k.oc;
      if (k.nout == 2 && ((E.ldr | E.roff | k.oc) & 1) == 0) {
        const float2 q2 = *reinterpret_cast<const float2*>(rp);
        in.r[h][0] = q2.x; in.r[h][1] = q2.y;
      } else {
        in.r[h][0] = rp[0];
        if (k.nout > 1) in.r[h][1] = rp[1];
      }
    }
  }
  return in;
}
// The arithmetic and the stores of column pair `k` in output row `orow`, whose loads have landed: bias b, cond c, residual
// r; v0 / v1 = the accumulator (or the split-K sum).  (alpha and the residual are an explicit multiply and add, never one
// fused multiply-add.)
__device__ __forceinline__ void tc_epi_store(const TcEpi& E, const TcEpiCol& k, long orow, float b0, float b1, float c0, float c1,
                                             float r0, float r1, float v0, float v1) {
  const float bv0 = E.cond ? b0 + c0 : b0, bv1 = E.cond ? b1 + c1 : b1;
  float u[2];
  if (E.gate) {
    const float a = v0 + bv0, s = v1 + bv1;
    u[0] = tanhf(a) * (1.f / (1.f + expf(-s)));
    u[1] = 0.f;
  } else {
    u[0] = v0 + bv0;
    u[1] = k.nout > 1 ? v1 + bv1 : 0.f;
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    float q = u[e];
    if (E.relu) q = fmaxf(q, 0.f);
    u[e] = __fmul_rn(q, E.alpha);
  }
  if (E.res) {
    u[0] = __fadd_rn(u[0], r0);
    if (k.nout > 1) u[1] = __fadd_rn(u[1], r1);
  }
  if (!E.store) return;
  const int oc = k.oc, nout = k.nout;
  if (E.y) {
    float* yr = E.y + orow * (long)E.ldy + E.yoff + oc;
    if (nout == 2 && ((E.ldy | E.yoff | oc) & 1) == 0) {
      *reinterpret_cast<float2*>(yr) = make_float2(u[0], u[1]);
    } else {
      yr[0] = u[0];
      if (nout > 1) yr[1] = u[1];
    }
  }
  if (E.p_hi) {
    const long po = orow * (long)E.ldp + E.poff + oc;
    __nv_bfloat16 hb[2], mb[2], lb[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float q = u[e];
      q = q > 0.f ? q : q * E.pl_slope;
      if (E.p_mid) split_bf16_3(q, hb[e], mb[e], lb[e]);
      else split_bf16(q, hb[e], lb[e]);
    }
    if (nout == 2 && ((E.ldp | E.poff | oc) & 1) == 0) {
      *reinterpret_cast<__nv_bfloat162*>(E.p_hi + po) = __halves2bfloat162(hb[0], hb[1]);
      *reinterpret_cast<__nv_bfloat162*>(E.p_lo + po) = __halves2bfloat162(lb[0], lb[1]);
      if (E.p_mid) *reinterpret_cast<__nv_bfloat162*>(E.p_mid + po) = __halves2bfloat162(mb[0], mb[1]);
    } else {
      E.p_hi[po] = hb[0]; E.p_lo[po] = lb[0];
      if (E.p_mid) E.p_mid[po] = mb[0];
      if (nout > 1) {
        E.p_hi[po + 1] = hb[1]; E.p_lo[po + 1] = lb[1];
        if (E.p_mid) E.p_mid[po + 1] = mb[1];
      }
    }
  }
}

template <int BN>
constexpr int tc_smem_bytes(int a_bytes, int np = 2, int ast = tc_ast<BN>(), int wst = tc_wst<BN>()) {
  return ast * np * a_bytes + wst * np * BN * TC_BK * 2 + 1024 /*alignment slack*/ + 256 /*barriers*/;
}
constexpr int TC_MAXST = 4;   // barrier slots per ring

// One output tile of a launch: 128 rows x BN channels of problem `P` in utterance `b`.
struct TcTile {
  int pi;           // problem index (the problem is always addressed as tb.p[pi]: a pointer into the __grid_constant__ parameter
                    //  turns every field access into a generic load instead of an indexed constant-bank read)
  int b, co0, t0, sp;
  int s;            // CTAs reducing this tile (split-K), sp = this CTA's rank among them
  int t0u;         // first row of the scheduling unit (== t0, or the pair's first tile with weight multicast)
  bool valid;       // the problem has this channel tile (grouped problems may differ in Cout)
};

// ---------------------------------------------------------------------------------------------------------------------
// The kernel body.  Launch shapes: (1) one tile per CTA, grid (row tiles, channel tiles, utterances x problems x split):
// the latency-bound single-utterance launches, with cluster split-K.  (2) tb.persist: a 1-D grid of one CTA per SM walks
// the same tile space with a stride of gridDim.x; the operand rings and their parities run on across tiles, so the
// producer fetches tile i+1's operands while the consumers run tile i's epilogue, and the per-CTA prologue (barrier
// init, descriptor prefetch, pipeline fill) is paid once per SM instead of once per tile.
// ---------------------------------------------------------------------------------------------------------------------
// MIXED: the single-wave image, which also runs mixed-split launches (tb.mixed); the persistent image never does (mixed
// splits imply split-K, and split-K launches are single-wave), so it is compiled without that code.
template <int BN, bool MIXED, class PT, int MP>
__device__ __forceinline__ void conv_tc_body(const TcBatchT<PT, MP>& tb, const int* __restrict__ lens, const int* __restrict__ offs) {
  constexpr bool HAS_MID = std::is_same<PT, TcProblem>::value;
  constexpr int B_BYTES = BN * TC_BK * 2;
  constexpr int NACC = BN / 2;                 // accumulator registers per consumer thread (m64nBN fragment)
  const int TC_AST = tb.ast, TC_WST = tb.wst, NP = HAS_MID ? tb.np : 2;
  PDL_LAUNCH();
  if (threadIdx.x == 0) TC_STAMP(0);
  const int S = tb.split;
  const bool persist = tb.persist != 0;
  const int A_BYTES = tb.a_bytes;
  const bool tall = tb.tall != 0;
  const int wmc = persist ? tb.wmc : 1;                    // CTAs sharing each weight tile (scheduling unit = wmc adjacent row tiles)
  const uint32_t wrank = wmc > 1 ? cluster_rank() : 0u;
  const int gxu = (tb.gx + wmc - 1) / wmc;
  const int ntiles = persist ? gxu * tb.gy * tb.gz : 1;
  const int tstride = persist ? (int)gridDim.x / wmc : 1;
  const int tile0 = persist ? (int)blockIdx.x / wmc : 0;
  // mixed-split launches: output tile `g` of this CTA's cluster, or the CTA's own tile (g < 0: g = rank / p.split)
  auto decode_mixed = [&](int g) {
    const int ci = (int)blockIdx.z / S, rank = (int)blockIdx.z - ci * S;
    int pi = 0;
    while (pi + 1 < tb.n && ci >= tb.p[pi + 1].cl0) ++pi;
    const int s = tb.p[pi].split, gyp = (tb.p[pi].Cout + BN - 1) / BN;
    if (g < 0) g = rank / s;
    const int tile = (ci - tb.p[pi].cl0) * (S / s) + g;
    TcTile t;
    t.pi = pi;
    t.s = s;
    t.sp = rank % s;
    t.t0 = (tile % tb.gx) * TC_BM;
    t.t0u = t.t0;
    t.co0 = ((tile / tb.gx) % gyp) * BN;
    t.b = tile / (tb.gx * gyp);
    t.valid = t.b < tb.nb;
    return t;
  };
  auto decode = [&](int tile) {
    if constexpr (MIXED) { if (tb.mixed) return decode_mixed(-1); }
    int bx, by, bz, bxu;
    if (persist) {
      bxu = tile % gxu;
      const int r = tile / gxu;
      by = r % tb.gy;
      bz = r / tb.gy;
      bx = bxu * wmc + (int)wrank;
    } else {
      bx = blockIdx.x; by = blockIdx.y; bz = blockIdx.z;
      bxu = bx;
    }
    TcTile t;
    t.t0u = bxu * wmc * TC_BM;
    const int zi = bz / S;
    t.s = S;
    t.sp = bz - zi * S;
    t.pi = zi % tb.n;
    t.b = zi / tb.n;
    t.co0 = by * BN;
    t.t0 = bx * TC_BM;
    t.valid = t.co0 < tb.p[t.pi].Cout;
    return t;
  };

  extern __shared__ uint8_t tc_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* smem_w = smem + TC_AST * NP * A_BYTES;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem_w + TC_WST * NP * B_BYTES);
  uint64_t* a_empty = a_full + TC_MAXST;
  uint64_t* w_full = a_empty + TC_MAXST;
  uint64_t* w_empty = w_full + TC_MAXST;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool producer = warp == TC_CWG * 4;
  const TcTile first = decode(tile0);
  const int cn = tb.cn;

  if (producer && lane == 0) {
    // every consumer warpgroup of every CTA reading a slot releases it
    for (int s = 0; s < TC_AST; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], (uint32_t)(cn * TC_CWG)); }
    for (int s = 0; s < TC_WST; ++s) { mbar_init(&w_full[s], 1); mbar_init(&w_empty[s], (uint32_t)(wmc * TC_CWG)); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    for (int q = 0; q < (persist ? tb.n : 1); ++q) {
      const PT& Q = tb.p[persist ? q : first.pi];
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&Q.a_hi)) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&Q.a_lo)) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&Q.w_hi)) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&Q.w_lo)) : "memory");
      if constexpr (HAS_MID) {
        if (NP == 3) {
          asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&Q.a_mid)) : "memory");
          asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&Q.w_mid)) : "memory");
        }
      }
    }
  }
  __syncthreads();
  const uint32_t crank = cn > 1 ? cluster_rank() : 0u;
  const uint16_t cmask = (uint16_t)((1u << cn) - 1u);
  if (cn > 1 || wmc > 1) cluster_sync_all();   // every peer's mbarriers exist before anybody multicasts into / arrives on them
  // Weights are immutable: the first ring of weight tiles is requested before waiting for the producer of the activations.
  // (lens/offs are final before any graph that reads them starts -- host copies or the previous phase's graph -- so the
  //  peek below only decides whether prefetching is worth it: idle CTAs of ragged batches must not fetch and then drain
  //  weights; the authoritative read stays after the wait)
  int w_pre = 0;
  auto issue_w = [&](const PT& P, int co0, int c, int j, int wst) {
    uint8_t* wb = smem_w + wst * NP * B_BYTES;
    mbar_expect_tx(&w_full[wst], NP * B_BYTES);
    if (wmc > 1) {
      // this CTA fetches channel rows [wrank, wrank + 1) * BN/2 of the tile and multicasts them into both CTAs of the pair;
      // the other half arrives from the peer and signals the same barrier
      const int half = (int)wrank * (BN / 2);
      tma_load_2d_mc(wb + half * 128, &P.w_hi, c * TC_BK, j * P.Cout + co0 + half, &w_full[wst], (uint16_t)3);
      tma_load_2d_mc(wb + B_BYTES + half * 128, &P.w_lo, c * TC_BK, j * P.Cout + co0 + half, &w_full[wst], (uint16_t)3);
      return;
    }
    tma_load_2d(wb, &P.w_hi, c * TC_BK, j * P.Cout + co0, &w_full[wst]);
    tma_load_2d(wb + B_BYTES, &P.w_lo, c * TC_BK, j * P.Cout + co0, &w_full[wst]);
    if constexpr (HAS_MID) { if (NP == 3) tma_load_2d(wb + 2 * B_BYTES, &P.w_mid, c * TC_BK, j * P.Cout + co0, &w_full[wst]); }
  };
  if (!persist && first.valid) {
    const PT& P = tb.p[first.pi];
    const int nsteps_all = (P.Cin / TC_BK) * P.k;
    const int s_beg = (int)((long)nsteps_all * first.sp / first.s), s_end = (int)((long)nsteps_all * (first.sp + 1) / first.s);
    const bool peek_active = first.t0 < lens[first.b] * tb.rmul + P.in_extra;
    w_pre = (tb.wpre && peek_active) ? min(TC_WST, s_end - s_beg) : 0;
    if (producer && lane == 0) {
      int c = s_beg / P.k, j = s_beg - c * P.k;
      for (int i = 0; i < w_pre; ++i) {          // w_pre <= TC_WST: slot == i
        issue_w(P, first.co0, c, j, i);
        if (++j == P.k) { j = 0; ++c; }
      }
    }
  }
  // everything above touched only this CTA's resources and constants; from here on the producer kernel's results are needed
  PDL_WAIT();
  if (threadIdx.x == 0) TC_STAMP(1);
  bool any_active = false;               // (split-K: the single tile of this CTA is active)

  if (producer) {
    // ------------------------------------------------------------------ TMA producer (one thread)
    // (ring slots, use parities and the (chunk, tap) pair of a k-step are carried as counters: the ring depths are launch
    //  parameters, and run-time divisions in the single producer thread are on the critical path of every step)
    if (lane == 0) {
      int ast = 0, a_use = 0, wst = 0, w_use = 0;    // ring slot / times the ring wrapped: run on across tiles
      for (int tile = tile0; tile < ntiles; tile += tstride) {
        const TcTile T = persist ? decode(tile) : first;
        if (!T.valid) continue;
        const PT& P = tb.p[T.pi];
        const int L = lens[T.b] * tb.rmul + P.in_extra;
        if (T.t0u >= L) {
          // nothing to compute; prefetched weight tiles must have landed before this CTA's shared memory is released
          for (int i = 0; i < w_pre; ++i) mbar_wait(&w_full[i], 0);
          continue;
        }
        any_active = true;
        const long in_base = (long)offs[T.b] * tb.rmul + (long)T.b * P.in_extra;
        const int nsteps_all = (P.Cin / TC_BK) * P.k;
        const int s_beg = (int)((long)nsteps_all * T.sp / T.s), s_end = (int)((long)nsteps_all * (T.sp + 1) / T.s);   // this CTA's k-steps
        const int a_per = tall ? P.k : 1;                    // k-steps sharing one activation tile (tall => S == 1)
        const uint32_t a_tx = (uint32_t)NP * (uint32_t)(tall ? (TC_BM + (P.k - 1) * P.dil) : TC_BM) * 128u;   // bytes TMA delivers per set of planes
        int c = s_beg / P.k, j = s_beg - c * P.k;
        int a_cnt = 0;                                         // steps since the last A tile
        for (int s = s_beg; s < s_end; ++s) {
          const int ls = s - s_beg;
          if (a_cnt == 0) {
            if (a_use > 0) mbar_wait(&a_empty[ast], (a_use - 1) & 1);
            uint8_t* ab = smem + ast * NP * A_BYTES;
            mbar_expect_tx(&a_full[ast], a_tx);
            const int row = (int)in_base + T.t0 - P.pad + (tall ? 0 : j * P.dil);
            if (cn > 1) {
              // this CTA fetches rows [crank, crank+1) * 128/cn of the tile and multicasts them to all cn CTAs
              const int slice = TC_BM / cn;
              const int soff = (int)crank * slice;
              tma_load_2d_mc(ab + soff * 128, &P.a_hi, c * TC_BK, row + soff, &a_full[ast], cmask);
              tma_load_2d_mc(ab + A_BYTES + soff * 128, &P.a_lo, c * TC_BK, row + soff, &a_full[ast], cmask);
            } else {
              tma_load_2d(ab, &P.a_hi, c * TC_BK, row, &a_full[ast]);
              tma_load_2d(ab + A_BYTES, &P.a_lo, c * TC_BK, row, &a_full[ast]);
              if constexpr (HAS_MID) { if (NP == 3) tma_load_2d(ab + 2 * A_BYTES, &P.a_mid, c * TC_BK, row, &a_full[ast]); }
            }
            if (++ast == TC_AST) { ast = 0; ++a_use; }
          }
          if (++a_cnt == a_per) a_cnt = 0;
          if (ls >= w_pre) {                                     // (the first ring was requested before PDL_WAIT)
            if (w_use > 0) mbar_wait(&w_empty[wst], (w_use - 1) & 1);
            issue_w(P, T.co0, c, j, wst);
          }
          if (++wst == TC_WST) { wst = 0; ++w_use; }
          if (++j == P.k) { j = 0; ++c; }
          if (ls == 0) TC_STAMP(2);
        }
        w_pre = 0;
        TC_STAMP(3);
      }
    }
    any_active = __shfl_sync(0xffffffffu, (int)any_active, 0) != 0;
  } else {
    // ------------------------------------------------------------------ consumers: wgmma mainloop + epilogue
    const int wg = warp >> 2;                              // rows [64 wg, 64 wg + 64) of the tile
    const int g = lane >> 2, q4 = lane & 3;
    const int rbase = wg * 64 + (warp & 3) * 16 + g;       // this thread's rows: rbase, rbase + 8
    const bool leader = (threadIdx.x & 127) == 0;
    int ast = 0, a_use = 0, wst = 0, w_use = 0;
    for (int tile = tile0; tile < ntiles; tile += tstride) {
      const TcTile T = persist ? decode(tile) : first;
      if (!T.valid) continue;
      const PT& P = tb.p[T.pi];
      const int L = lens[T.b] * tb.rmul + P.in_extra;
      if (T.t0u >= L) continue;                              // (with weight multicast a CTA whose own tile lies behind the end of the
                                                             //  utterance still runs the mainloop; it stores nothing)
      any_active = true;
      const int nsteps_all = (P.Cin / TC_BK) * P.k;
      const int s_beg = (int)((long)nsteps_all * T.sp / T.s), s_end = (int)((long)nsteps_all * (T.sp + 1) / T.s);
      const int a_per = tall ? P.k : 1;
      float acc[NACC];
#pragma unroll
      for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
      int j = s_beg % P.k;
      int a_cnt = 0;
      // the slots of the previous k-step are released once its MMAs have retired (one wgmma group stays in flight)
      int prev_w = -1, prev_a = -1;
      for (int s = s_beg; s < s_end; ++s) {
        const int ls = s - s_beg;
        if (a_cnt == 0) mbar_wait(&a_full[ast], a_use & 1);
        mbar_wait(&w_full[wst], w_use & 1);
        if (ls == 0 && threadIdx.x == 0) TC_STAMP(4);
        const uint32_t abase = smem_u32(smem + ast * NP * A_BYTES) + (uint32_t)(wg * 64 * 128) + (tall ? (uint32_t)(j * P.dil) * 128u : 0u);
        const uint32_t wbase = smem_u32(smem_w + wst * NP * B_BYTES);
        const uint64_t ahi = gmma_desc_sw128(abase, tb.baseoff), alo = gmma_desc_sw128(abase + A_BYTES, tb.baseoff);
        const uint64_t bhi = gmma_desc_sw128(wbase), blo = gmma_desc_sw128(wbase + B_BYTES);
        auto mma = [&](uint64_t da, uint64_t db) {
          if constexpr (BN == 128) wgmma_ss_n128(acc, da, db);
          else wgmma_ss_n64(acc, da, db);
        };
        wgmma_fence();
        if (tb.dbgskip & 2) {
        } else if (NP == 3) {
          // exact 3-way split: the six products that reach the last bit of an fp32 product, smallest first
          const uint64_t ami = gmma_desc_sw128(abase + 2 * A_BYTES, tb.baseoff), bmi = gmma_desc_sw128(wbase + 2 * B_BYTES);
#pragma unroll
          for (int kk = 0; kk < TC_BK / 16; ++kk) {
            const uint64_t adv = (uint64_t)((kk * 32) >> 4);
            mma(ahi + adv, blo + adv);
            mma(alo + adv, bhi + adv);
            mma(ami + adv, bmi + adv);
            mma(ami + adv, bhi + adv);
            mma(ahi + adv, bmi + adv);
            mma(ahi + adv, bhi + adv);
          }
        } else {
#pragma unroll
          for (int kk = 0; kk < TC_BK / 16; ++kk) {
            const uint64_t adv = (uint64_t)((kk * 32) >> 4);     // 16 bf16 = 32 bytes along K inside the swizzle atom
            mma(alo + adv, bhi + adv);
            mma(ahi + adv, blo + adv);
            mma(ahi + adv, bhi + adv);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        wgmma_touch<NACC>(acc);
        if (leader) {
          if (prev_w >= 0) tc_release(&w_empty[prev_w], wmc);
          if (prev_a >= 0) tc_release(&a_empty[prev_a], cn);
        }
        prev_w = wst;
        prev_a = -1;
        if (++wst == TC_WST) { wst = 0; ++w_use; }
        if (++a_cnt == a_per) {                                // the activation tile is released after its last tap
          prev_a = ast;
          a_cnt = 0;
          if (++ast == TC_AST) { ast = 0; ++a_use; }
        }
        if (++j == P.k) j = 0;
      }
      // ---- epilogue.  This thread finishes the column pairs j = 0 .. W/8 - 1 of the tile's columns [co0 + sp W, + W) that
      // its CTA owns (W = BN unsplit): columns 8 j + 2 q4 of rows rbase and rbase + 8.  Unsplit, pair j of row h is the
      // accumulator pair (acc[4j + 2h], acc[4j + 2h + 1]).  The loops are not unrolled, so the epilogue is one copy of its
      // code: unrolled over a tile's pairs it ran once per CTA from a cold instruction cache and cost 6-12 us of every
      // split-K launch (CTA 0 stamps, tools/decoder_phases.py).
      const int W = BN / T.s, ncp = W / 8;
      const TcEpi E = tc_epi(P, T.b, tb.dbgskip);
      const int cbase = T.co0 + T.sp * W + 2 * q4;
      long orow[2];
      bool rowok[2];
      {
        const long out_base = (long)offs[T.b] * tb.rmul * P.out_mul + (long)T.b * P.out_seq_extra;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int t = T.t0 + rbase + 8 * h;
          rowok[h] = t < L;
          orow[h] = out_base + (long)t * P.out_mul + P.out_add;
        }
      }
      auto col = [&](int j) { return tc_epi_col(E, cbase + 8 * j, j < ncp); };
      // the first pair's loads go out before the last MMAs retire (and before the split-K cluster barriers)
      TcEpiIn in = tc_epi_load(E, col(0), orow, rowok);
      wgmma_wait<0>();
      wgmma_touch<NACC>(acc);
      if (leader) {
        if (prev_w >= 0) tc_release(&w_empty[prev_w], wmc);
        if (prev_a >= 0) tc_release(&a_empty[prev_a], cn);
      }
      if (threadIdx.x == 0) TC_STAMP(5);
      float* stage = reinterpret_cast<float*>(smem);         // split-K: [T.s][128][W] fp32 (BN/2 KB), aliases the operand rings
      if (T.s > 1) {
        // split-K reduce-scatter among the T.s ranks g0 .. g0 + T.s - 1 of the tile: rank g0 + q finishes columns [q W, q W + W).
        // Every CTA sends each partial pair to the owner's staging buffer [src][row][W]; the owner adds the partials in rank order.
        const int sp = T.sp, g0 = MIXED ? (int)blockIdx.z % S - sp : 0;
        cluster_sync_all();                                  // (1) every CTA of the cluster is done with its operand rings
#pragma unroll
        for (int jn = 0; jn < BN / 8; ++jn) {
          const int cc = jn * 8 + 2 * q4;
          const int qo = cc / W;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint32_t ra;
            asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(smem_u32(stage + ((size_t)sp * TC_BM + rbase + 8 * h) * W + (cc - qo * W))), "r"(g0 + qo));
            asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(ra), "f"(acc[4 * jn + 2 * h]), "f"(acc[4 * jn + 2 * h + 1]) : "memory");
          }
        }
        cluster_sync_all();                                  // (2) all partials have landed; nobody writes into a CTA after this point
      }
#pragma unroll 1
      for (int j = 0; j < ncp; ++j) {
        const TcEpiIn nx = tc_epi_load(E, col(j + 1), orow, rowok);   // the next pair's loads, ahead of this pair's stores
        const TcEpiCol k = col(j);
        // one row at a time, so the code of a (row, column pair) exists once: with both rows inlined the 128-wide images
        // spill at their register limit (168 = 64K / (3 warps per SM sub-partition x 32 x 4))
#pragma unroll 1
        for (int h = 0; h < 2; ++h) {
          if (!k.ok || !(h ? rowok[1] : rowok[0])) continue;
          float v0 = h ? acc[2] : acc[0], v1 = h ? acc[3] : acc[1];
          if (T.s > 1) {                                     // the owner's sum of the partials, in rank order
            const float* st = stage + (size_t)(rbase + 8 * h) * W + 8 * j + 2 * q4;
            v0 = 0.f; v1 = 0.f;
#pragma unroll 1
            for (int src = 0; src < T.s; ++src) {
              const float2 p2 = *reinterpret_cast<const float2*>(st + (size_t)src * TC_BM * W);
              v0 += p2.x; v1 += p2.y;
            }
          }
          tc_epi_store(E, k, h ? orow[1] : orow[0], in.b0, in.b1, in.c0, in.c1, h ? in.r[1][0] : in.r[0][0],
                       h ? in.r[1][1] : in.r[0][1], v0, v1);
        }
        // the next pair's accumulators move to the front (static register indices in a loop that is not unrolled)
#pragma unroll
        for (int i = 0; i + 4 < NACC; ++i) acc[i] = acc[i + 4];
        in = nx;
      }
    }
  }
  if (first.s > 1) {
    // every CTA of a cluster with an active tile takes part in the two split-K cluster barriers: the producer warp always,
    // the consumers here when their own tile is idle (mixed-split clusters cover several tiles, not all of them active)
    bool cl_active = any_active;
    if (MIXED && tb.mixed)
      for (int g = 0; g < S / first.s; ++g) {
        const TcTile u = decode_mixed(g);
        if (u.valid && u.t0 < lens[u.b] * tb.rmul + tb.p[u.pi].in_extra) cl_active = true;
      }
    if (cl_active && (producer || !any_active)) {
      __syncwarp();
      cluster_sync_all();
      cluster_sync_all();
    }
  }
  if (threadIdx.x == 0) TC_STAMP(7);
  __syncthreads();
  if (cn > 1 || wmc > 1) cluster_sync_all();   // no peer may still multicast into, or arrive on, this CTA's shared memory
  if (threadIdx.x == 0) TC_STAMP(8);
}

// Single-wave launches (cluster split-K, or one tile per CTA).  DYN = false: two operand planes, the launch descriptor without
// the third-plane tensor maps (the default single-utterance launches).
template <int BN, bool DYN, int MP = TC_MAXP>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_kernel(const __grid_constant__ TcBatchT<std::conditional_t<DYN, TcProblem, TcProblemBase>, MP> tb, const int* __restrict__ lens,
               const int* __restrict__ offs) {
  conv_tc_body<BN, true>(tb, lens, offs);
}
// More than one wave of tiles: persistent grid (tb.persist), or one tile per CTA.
template <int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_persist_kernel(const __grid_constant__ TcBatch tb, const int* __restrict__ lens, const int* __restrict__ offs) {
  conv_tc_body<BN, false>(tb, lens, offs);
}

// ------------------------------------------------------------------------------------------------
// fp32 rows -> split-bf16 planes (optionally through leaky-relu and the ReflectionPad1d((1,0)) row shift of
// models.py:1039) for tensors that were not produced by a tensor-core epilogue.
// ------------------------------------------------------------------------------------------------
// Row blocking of the elementwise plane kernels: a block of EW_THREADS threads covers EW_ROWS consecutive rows of one
// utterance, C/4 threads per row (one block per row left most of a batched launch in block-scheduling overhead:
// mrf_mean_planes 8.1 ms of a 70 ms batch-64 step, profiles/r2_launches_batch64.csv).
constexpr int EW_THREADS = 256;
constexpr int EW_ROWS = 16;

__global__ void __launch_bounds__(EW_THREADS)
split_planes_kernel(const float* __restrict__ x, int ldx, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                    int ldp, int C, float slope, int reflect, int rmul, const int* __restrict__ lens,
                    const int* __restrict__ offs) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y;
  const int Lphys = lens[b] * rmul;
  const int L = Lphys + (reflect ? 1 : 0);
  const int p0 = blockIdx.x * EW_ROWS;
  if (p0 >= L) return;
  const int nq = C >> 2;                               // float4 units per row
  const int nrow = min(EW_ROWS, L - p0);
  const long base = (long)offs[b] * rmul;
  for (int u = threadIdx.x; u < nrow * nq; u += EW_THREADS) {
    const int r = u / nq, c = (u - r * nq) << 2;
    const int p = p0 + r;
    const int pr = reflect ? (p == 0 ? 1 : p - 1) : p;
    const long irow = base + pr;
    const long orow = base + (reflect ? b : 0) + p;
    const float4 v = *reinterpret_cast<const float4*>(x + irow * ldx + c);
    const float f[4] = {v.x, v.y, v.z, v.w};
    __align__(8) __nv_bfloat16 hb[4], lb[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float q = f[i] > 0.f ? f[i] : f[i] * slope;
      split_bf16(q, hb[i], lb[i]);
    }
    *reinterpret_cast<uint2*>(hi + orow * ldp + c) = *reinterpret_cast<const uint2*>(hb);
    *reinterpret_cast<uint2*>(lo + orow * ldp + c) = *reinterpret_cast<const uint2*>(lb);
  }
}

// mean of the resblock outputs of an MRF stage (models.py: xs / num_kernels) -> fp32 rows (optional) + planes of lrelu(mean)
__global__ void __launch_bounds__(EW_THREADS)
mrf_mean_planes_kernel(const float* __restrict__ a, const float* __restrict__ b2, const float* __restrict__ c3, int n,
                       float* __restrict__ out, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int C,
                       float slope, int reflect, int rmul, const int* __restrict__ lens, const int* __restrict__ offs) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y;
  const int Lphys = lens[b] * rmul;
  const int L = Lphys + (reflect ? 1 : 0);
  const int p0 = blockIdx.x * EW_ROWS;
  if (p0 >= L) return;
  const int nq = C >> 2;
  const int nrow = min(EW_ROWS, L - p0);
  const long base = (long)offs[b] * rmul;
  const float d = (float)n;
  for (int u = threadIdx.x; u < nrow * nq; u += EW_THREADS) {
    const int r = u / nq, c = (u - r * nq) << 2;
    const int p = p0 + r;
    const int pr = reflect ? (p == 0 ? 1 : p - 1) : p;
    const long irow = base + pr;
    const long orow = base + (reflect ? b : 0) + p;
    float4 s = *reinterpret_cast<const float4*>(a + irow * C + c);
    if (n > 1) { const float4 q = *reinterpret_cast<const float4*>(b2 + irow * C + c); s.x += q.x; s.y += q.y; s.z += q.z; s.w += q.w; }
    if (n > 2) { const float4 q = *reinterpret_cast<const float4*>(c3 + irow * C + c); s.x += q.x; s.y += q.y; s.z += q.z; s.w += q.w; }
    s.x /= d; s.y /= d; s.z /= d; s.w /= d;
    if (out && (!reflect || p >= 1)) *reinterpret_cast<float4*>(out + irow * C + c) = s;
    const float f[4] = {s.x, s.y, s.z, s.w};
    __align__(8) __nv_bfloat16 hb[4], lb[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float q = f[i] > 0.f ? f[i] : f[i] * slope;
      split_bf16(q, hb[i], lb[i]);
    }
    *reinterpret_cast<uint2*>(hi + orow * C + c) = *reinterpret_cast<const uint2*>(hb);
    *reinterpret_cast<uint2*>(lo + orow * C + c) = *reinterpret_cast<const uint2*>(lb);
  }
}

}  // namespace vtts
