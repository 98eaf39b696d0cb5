// kernels.cuh -- hand-written sm_90a kernels of the VITS2 inference path (fp32 FFMA family).
//
// Activation layout: channels-last, packed utterances.  A tensor that the reference holds as
// [B, C, T] (training/vits2/models.py) lives here as rows[off[b] + t][C]; `len[b]`/`off[b]` are
// device arrays so that the frame-resolution kernels never need the host to know T_y.
// Positions outside [0, len) are never written and read as zero, which reproduces both the
// reference's x_mask multiplications (attentions.py:50,298,301; modules.py:96-108,148-176) and the
// per-utterance zero padding of the unmasked decoder convs (modules.py:210-225 with x_mask=None).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

namespace vtts {

// Programmatic dependent launch (PDL): every kernel of the engine is launched with programmatic stream serialisation,
// so kernel N+1 may start (and run its prologue: barrier init, weight prefetch) while kernel N drains.
// PDL_WAIT() blocks until the predecessor grid has completed and its writes are visible; nothing that a predecessor
// produces (activations, lens/offs) may be touched, and nothing may be written, before it.  Both are no-ops when the
// kernel was launched without the attribute.
// Optional in-graph timeline (tools/timeline.py): CTA (0,0,0) of every kernel appends (source line, %globaltimer) at entry.
__device__ unsigned long long* g_timeline = nullptr;     // [0] = counter, then pairs (line, ns)
__device__ __forceinline__ void timeline_stamp(int line) {
  unsigned long long* tl = g_timeline;
  if (tl && threadIdx.x == 0 && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    const unsigned long long i = atomicAdd(tl, 1ull);
    if (i < 4000) { tl[1 + 2 * i] = (unsigned long long)line; tl[2 + 2 * i] = t; }
  }
}
// The trigger comes AFTER the wait: a kernel that triggered at entry would let its successor start, trigger in turn, and
// so on -- inside a CUDA graph the whole chain piles onto the SMs spinning in griddepcontrol.wait (measured: slower).
// Triggering after the wait keeps exactly one successor in flight: its launch latency and prologue overlap this
// kernel's main work.
// same, for one designated thread of CTA (0,0,0) that is not thread 0 (warp-specialised kernels)
__device__ __forceinline__ void timeline_stamp_t(int line) {
  unsigned long long* tl = g_timeline;
  if (tl && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    const unsigned long long i = atomicAdd(tl, 1ull);
    if (i < 4000) { tl[1 + 2 * i] = (unsigned long long)line; tl[2 + 2 * i] = t; }
  }
}
#define PDL_LAUNCH() timeline_stamp(__LINE__)
#define PDL_WAIT() asm volatile("griddepcontrol.wait;\n\tgriddepcontrol.launch_dependents;" ::: "memory")

// ---- mbarrier / bulk-async-copy wrappers (shared by the tensor-core conv and the DDS kernel)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra.uni WAIT_DONE;\n"
      "bra.uni WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 1-D bulk async copy global -> shared (TMA engine, no tensor map); completion is signalled on an mbarrier
__device__ __forceinline__ void bulk_copy_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// fp32 -> (hi, lo) bf16 with hi + lo == x to ~2^-18 relative: the operand format of the tensor-core convs.
// Rounding to bf16 is done on the bit pattern (add half an ulp of the kept part, drop the low 16 bits: round to nearest,
// ties away from zero) instead of cvt.rn.bf16.f32: the conversion pipe runs at a quarter of the integer / FP32 rate, and
// every tensor-core epilogue converts two values per output element (ncu/timeline: ~0.5 us of a 2.4 us epilogue).
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  const uint32_t h = (__float_as_uint(x) + 0x8000u) & 0xFFFF0000u;
  const float r = x - __uint_as_float(h);                 // exact
  const uint32_t l = __float_as_uint(r) + 0x8000u;
  hi = __ushort_as_bfloat16((unsigned short)(h >> 16));
  lo = __ushort_as_bfloat16((unsigned short)(l >> 16));
}
// fp32 -> (hi, mid, lo) bf16 with hi + mid + lo == x EXACTLY up to the last bit of the fp32 significand (3 x 8 = 24 bits):
// with the six products hh, hm, mh, hl, lh, mm a tensor-core GEMM then multiplies like an fp32 FMA pipe does (the dropped
// terms ml, lm, ll are below 2^-26 of the product) and differs from it only in the fp32 summation order.  Used where the
// result feeds ceil() of a duration (text encoder, precision mode 3).
__device__ __forceinline__ void split_bf16_3(float x, __nv_bfloat16& hi, __nv_bfloat16& mid, __nv_bfloat16& lo) {
  const uint32_t h = (__float_as_uint(x) + 0x8000u) & 0xFFFF0000u;
  const float r1 = x - __uint_as_float(h);
  const uint32_t m = (__float_as_uint(r1) + 0x8000u) & 0xFFFF0000u;
  const float r2 = r1 - __uint_as_float(m);
  const uint32_t l = __float_as_uint(r2) + 0x8000u;
  hi = __ushort_as_bfloat16((unsigned short)(h >> 16));
  mid = __ushort_as_bfloat16((unsigned short)(m >> 16));
  lo = __ushort_as_bfloat16((unsigned short)(l >> 16));
}
// two values at once, packed as bf16 pairs (a in the low half): PRMT does the packing
__device__ __forceinline__ void split_bf16_pair(float a, float b, uint32_t& hi, uint32_t& lo) {
  const uint32_t ha = (__float_as_uint(a) + 0x8000u) & 0xFFFF0000u, hb = (__float_as_uint(b) + 0x8000u) & 0xFFFF0000u;
  const uint32_t la = __float_as_uint(a - __uint_as_float(ha)) + 0x8000u, lb = __float_as_uint(b - __uint_as_float(hb)) + 0x8000u;
  hi = __byte_perm(ha, hb, 0x7632);
  lo = __byte_perm(la, lb, 0x7632);
}

// ------------------------------------------------------------------------------------------------
// Generic grouped conv1d-as-GEMM (direct, im2col-free), fp32 FFMA.
//   y[t*out_mul + out_add][co] = epi( bias[co] + cond[b][co] + sum_{j,ci} w[j][ci][co] * pro(x[t + j*dil - pad][ci]) )
// Covers every dense contraction of the path: 1x1 convs (attentions.py:156-162, models.py:374-386),
// FFN convs (attentions.py:294-302), WN in/res-skip layers (modules.py:155-175), conv_pre
// (models.py:1024), the polyphase branches of ConvTranspose1d (models.py:1027-1028), ResBlock convs
// (modules.py:210-225), conv_post (models.py:1040).
// ------------------------------------------------------------------------------------------------
constexpr int CV_TT = 64;        // time rows per CTA
constexpr int CV_TC = 64;        // output channels per CTA
constexpr int CV_CK = 16;        // input channels per k-step
constexpr int CV_THREADS = 128;  // 16 (time) x 8 (channel groups of 8)
constexpr int CV_MAXP = 4;       // problems per grouped launch
constexpr int CV_XR = 4;         // float4 registers per thread for the input-tile prefetch

enum : int { PRO_NONE = 0, PRO_LRELU = 1 };
enum : int { EPI_RELU = 1, EPI_GATE = 2, EPI_TANH = 4 };

struct ConvP {
  const float* x;     // input rows
  const float* w;     // [k][Cin][ldw]
  const float* bias;  // [ldw]
  const float* cond;  // per-utterance vector cond[b*cond_ld + co] added before the activation, or null
  const float* res;   // residual added after alpha scaling (same row indexing as y), or null
  float* y;
  int ldx, xoff, ldw, cond_ld, ldr, roff, ldy, yoff;
  int Cin, Cout, k, dil, pad;
  int in_extra;       // logical length = len*rmul + in_extra (ReflectionPad1d((1,0)), models.py:1039)
  int reflect;        // logical input p maps to physical row (p == 0 ? 1 : p - 1)
  int out_mul, out_add, out_seq_extra;
  int pro;
  float slope;
  int epi;
  float alpha;
  __nv_bfloat16* p_hi;   // optional split-bf16 planes of the output (same rows, `ldp` channels per row) for a
  __nv_bfloat16* p_lo;   // tensor-core consumer; written as lrelu(out, pl_slope)
  __nv_bfloat16* p_mid;  // third plane (exact 3-way split) or null
  int ldp;
  float pl_slope;
};

struct ConvBatch {
  int stage_off;   // float offset of the split-K staging buffer [S][8/S][128] float4 in dynamic shared memory
  ConvP p[CV_MAXP];
  int n;
  int rmul;  // rows per length unit of the input (1, 4, 16 ...)
  int xw;    // smem row pitch of the input tile (floats), == 1 (mod 8)
  int S;     // thread-block-cluster size along grid.x: the k-steps of a tile are split over S CTAs
};

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, int src_bytes) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gsrc), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// thread-block-cluster barrier (all threads of all CTAs) with release/acquire semantics
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}
// load a float from the shared memory of CTA `rank` of this cluster (distributed shared memory)
__device__ __forceinline__ float ld_dsmem(const float* local_smem_ptr, int rank) {
  unsigned la = (unsigned)__cvta_generic_to_shared(local_smem_ptr), ra;
  float v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(ra) : "r"(la), "r"(rank));
  asm volatile("ld.shared::cluster.f32 %0, [%1];\n" : "=f"(v) : "r"(ra) : "memory");
  return v;
}

// Work decomposition (one CTA = one 64(time) x 64(channel) output tile of one problem of one utterance):
//  * G thread groups of 128 split the 16*G input channels of every k-step (intra-CTA split-K);
//  * S CTAs of a thread-block cluster split the k-steps (s = rank, rank+S, ...) and reduce their partial
//    tiles through distributed shared memory in a fixed order (deterministic), each CTA finishing 1/S of
//    the tile.  At batch 1 a conv has only a handful of output tiles; the cluster dimension is what lets
//    it spread over the SMs.
//  * inside a group each thread accumulates 4 rows (tx + 16m) x 8 channels (shared-memory operand delivery is
//    128 B/clk/SM of *delivered* data, so wider register tiles than the 2x16 variant tried first are needed).
// Weight tiles run through an NS-deep cp.async ring (one __syncthreads per step); the input tile of the
// next needed channel chunk is prefetched into registers (prologue applied) and double-buffered.
constexpr int CV_NS = 3;

template <int G>
__global__ void __launch_bounds__(CV_THREADS * G)
conv_kernel(const __grid_constant__ ConvBatch cb, const int* __restrict__ lens, const int* __restrict__ offs) {
  constexpr int CKS = CV_CK * G;        // channels per step over all groups
  constexpr int NT = CV_THREADS * G;
  PDL_LAUNCH();
  const int S = cb.S;                   // cluster size along x (1, 2, 4, 8)
  const int rank = S > 1 ? (int)(blockIdx.x % S) : 0;
  const int pi = blockIdx.z % cb.n;
  const int b = blockIdx.z / cb.n;
  const ConvP& P = cb.p[pi];
  const int co0 = blockIdx.y * CV_TC;
  if (co0 >= P.Cout) return;            // uniform over the cluster
  const int t0 = (int)(blockIdx.x / S) * CV_TT;

  extern __shared__ __align__(16) float smem[];
  const int xw = cb.xw;
  float* Xs = smem;                      // [2][CKS][xw]
  float* Ws = smem + 2 * CKS * xw;       // [NS][CKS][TC]

  const int tid = threadIdx.x;
  const int grp = tid / CV_THREADS;
  const int ltid = tid - grp * CV_THREADS;
  const int tx = ltid & 15;              // time rows tx + 16*m
  const int ty = ltid >> 4;              // 8-channel strip
  const int k = P.k, dil = P.dil;
  const int n_pos = CV_TT + (k - 1) * dil;
  const int nchunks = P.Cin / CKS;
  const int nsteps = nchunks * k;
  // my steps: a contiguous range, so that the k taps of a channel chunk reuse one staged input tile
  const int s_beg = (int)((long)nsteps * rank / S), s_end = (int)((long)nsteps * (rank + 1) / S);
  const int nmine = s_end - s_beg;

  float acc[4][8];
#pragma unroll
  for (int m = 0; m < 4; ++m)
#pragma unroll
    for (int n = 0; n < 8; ++n) acc[m][n] = 0.f;

  float4 xr[CV_XR];
  int Lphys = 0, L = 0;                  // set after PDL_WAIT (lens/offs may come from a predecessor kernel)
  long in_base = 0, out_base = 0;

  auto load_x = [&](int c) {
#pragma unroll
    for (int e = 0; e < CV_XR; ++e) {
      const int it = tid + e * NT;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (it < n_pos * 4 * G) {
        const int pos = it / (4 * G);
        const int q = (it - pos * 4 * G) * 4;
        const int p = t0 + pos - P.pad;
        if (p >= 0 && p < L) {
          const int pr = P.reflect ? (p == 0 ? 1 : p - 1) : p;
          v = __ldg(reinterpret_cast<const float4*>(P.x + (in_base + pr) * (long)P.ldx + P.xoff + c * CKS + q));
          if (P.pro == PRO_LRELU) {
            v.x = v.x > 0.f ? v.x : v.x * P.slope;
            v.y = v.y > 0.f ? v.y : v.y * P.slope;
            v.z = v.z > 0.f ? v.z : v.z * P.slope;
            v.w = v.w > 0.f ? v.w : v.w * P.slope;
          }
        }
      }
      xr[e] = v;
    }
  };
  auto store_x = [&](int xb) {
    float* dst = Xs + xb * CKS * xw;
#pragma unroll
    for (int e = 0; e < CV_XR; ++e) {
      const int it = tid + e * NT;
      if (it < n_pos * 4 * G) {
        const int pos = it / (4 * G);
        const int q = (it - pos * 4 * G) * 4;
        dst[(q + 0) * xw + pos] = xr[e].x;
        dst[(q + 1) * xw + pos] = xr[e].y;
        dst[(q + 2) * xw + pos] = xr[e].z;
        dst[(q + 3) * xw + pos] = xr[e].w;
      }
    }
  };
  auto issue_w = [&](int i) {            // i-th of my steps
    const int s = s_beg + i;
    const int c = s / k, j = s - c * k;
    float* dst = Ws + (i % CV_NS) * CKS * CV_TC;
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int f = tid + e * NT;
      const int r = f >> 4;
      const int c4 = (f & 15) * 4;
      const bool ok = (co0 + c4) < P.ldw;
      const float* src = P.w + ((long)(j * P.Cin + c * CKS + r) * P.ldw + (ok ? co0 + c4 : 0));
      cp_async16(dst + r * CV_TC + c4, src, ok ? 16 : 0);
    }
  };

  // weights are immutable: their first tiles are requested before waiting for the producer of the activations
#pragma unroll
  for (int i = 0; i < CV_NS - 1; ++i) {
    if (i < nmine) issue_w(i);
    cp_async_commit();
  }
  PDL_WAIT();
  Lphys = lens[b] * cb.rmul;
  L = Lphys + P.in_extra;
  if (t0 >= L) return;                  // uniform over the cluster (pending cp.async into our own smem is harmless)
  // Distributed shared memory may only be touched once the owning CTA is known to be running: every CTA announces itself
  // here (non-blocking) and the matching wait sits right before the first remote store of the split-K reduction
  if (S > 1) asm volatile("barrier.cluster.arrive.relaxed.aligned;\n" ::: "memory");
  in_base = (long)offs[b] * cb.rmul;
  out_base = in_base * P.out_mul + (long)b * P.out_seq_extra;
  int xbuf = 0;        // Xs buffer holding the chunk of the current step
  bool pending = false; // xr holds the next chunk, not yet staged
  if (nmine > 0) {
    load_x(s_beg / k);
    store_x(0);
  }
  timeline_stamp(-21);
  for (int i = 0; i < nmine; ++i) {
    const int s = s_beg + i;
    const int c = s / k, j = s - c * k;
    // chunk needed by my next step (prefetch into registers while this step computes; fetching it earlier was measured slower)
    if (i + 1 < nmine && (s + 1) / k != c) { load_x((s + 1) / k); pending = true; }
    cp_async_wait<CV_NS - 2>();
    __syncthreads();                       // W[i] (and a freshly stored X chunk) visible; ring slot (i-1)%NS free
    if (i + CV_NS - 1 < nmine) issue_w(i + CV_NS - 1);
    cp_async_commit();
    const float* xs = Xs + (xbuf * CKS + grp * CV_CK) * xw + tx + j * dil;
    const float* ws = Ws + ((i % CV_NS) * CKS + grp * CV_CK) * CV_TC + ty * 8;
#pragma unroll
    for (int ci = 0; ci < CV_CK; ++ci) {
      float a[4];
#pragma unroll
      for (int m = 0; m < 4; ++m) a[m] = xs[ci * xw + 16 * m];
      const float4 b0 = *reinterpret_cast<const float4*>(ws + ci * CV_TC);
      const float4 b1 = *reinterpret_cast<const float4*>(ws + ci * CV_TC + 4);
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int m = 0; m < 4; ++m)
#pragma unroll
        for (int n = 0; n < 8; ++n) acc[m][n] = fmaf(a[m], bb[n], acc[m][n]);
    }
    if (pending && (s + 1) / k != c) {      // last tap of this chunk: stage the next one (that buffer was last read >= 1 barrier ago)
      store_x(xbuf ^ 1);
      xbuf ^= 1;
      pending = false;
    }
  }

  // ---- reductions: groups (shared memory) then cluster ranks (distributed shared memory), fixed order
  timeline_stamp(-22);
  cp_async_wait<0>();
  __syncthreads();
  float* red = smem;                                       // [G-1][32][128], aliases the (now idle) pipeline buffers
  if (G > 1) {
    if (grp > 0) {
#pragma unroll
      for (int m = 0; m < 4; ++m)
#pragma unroll
        for (int n = 0; n < 8; ++n) red[((grp - 1) * 32 + m * 8 + n) * CV_THREADS + ltid] = acc[m][n];
    }
    __syncthreads();
    if (grp == 0) {
#pragma unroll
      for (int g2 = 0; g2 < G - 1; ++g2)
#pragma unroll
        for (int m = 0; m < 4; ++m)
#pragma unroll
          for (int n = 0; n < 8; ++n) acc[m][n] += red[(g2 * 32 + m * 8 + n) * CV_THREADS + ltid];
    }
  }
  // A thread's 4 x 8 tile is 8 units of 4 channels (unit g = row m = g/2, half qh = g%2); unit g is finished by rank
  // g*S/8.  Every rank PUSHES its partial units into the owners' staging buffers [src rank][unit][thread] (a region no
  // pipeline buffer aliases, so peers still in their main loop are not disturbed); after one cluster barrier each owner
  // adds the S partials of its units in rank order.
  int m_lo = 0, m_hi = 4, q_lo = 0, q_hi = 2;
  if (S > 1) {
    const int ne4 = 8 / S;                                 // units per owner
    float4* stage = reinterpret_cast<float4*>(smem + cb.stage_off);
    asm volatile("barrier.cluster.wait.aligned;\n" ::: "memory");   // all peers have started (announced at kernel entry)
    if (grp == 0) {
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        const int owner = (g * S) >> 3, u = g & (ne4 - 1);
        const uint32_t la = smem_u32(stage + ((rank * ne4 + u) * CV_THREADS + ltid));
        uint32_t ra;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(la), "r"(owner));
        asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(ra), "f"(acc[g >> 1][(g & 1) * 4 + 0]),
                     "f"(acc[g >> 1][(g & 1) * 4 + 1]), "f"(acc[g >> 1][(g & 1) * 4 + 2]), "f"(acc[g >> 1][(g & 1) * 4 + 3])
                     : "memory");
      }
    }
    cluster_sync_all();                                    // all partials landed; nobody touches a peer after this
    if (S == 2) { m_lo = 2 * rank; m_hi = m_lo + 2; }
    else if (S == 4) { m_lo = rank; m_hi = rank + 1; }
    else { m_lo = rank >> 1; m_hi = m_lo + 1; q_lo = rank & 1; q_hi = q_lo + 1; }
    if (grp == 0) {
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        if (((g * S) >> 3) == rank) {
          const int u = g & (ne4 - 1);
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int r2 = 0; r2 < S; ++r2) {                 // fixed summation order
            const float4 q4 = stage[(r2 * ne4 + u) * CV_THREADS + ltid];
            v.x += q4.x; v.y += q4.y; v.z += q4.z; v.w += q4.w;
          }
          acc[g >> 1][(g & 1) * 4 + 0] = v.x; acc[g >> 1][(g & 1) * 4 + 1] = v.y;
          acc[g >> 1][(g & 1) * 4 + 2] = v.z; acc[g >> 1][(g & 1) * 4 + 3] = v.w;
        }
      }
    }
  }
  if (grp > 0) return;
  timeline_stamp(-23);

  // ---- epilogue on the owned units
  const int co = co0 + ty * 8;
  if (co >= P.Cout) return;
  const bool gate = (P.epi & EPI_GATE) != 0;
  const bool aligned = ((P.ldy | P.yoff) & 3) == 0 && (!P.res || ((P.ldr | P.roff) & 3) == 0);
  const int climit = gate ? (P.Cout >> 1) : P.Cout;
#pragma unroll
  for (int m = 0; m < 4; ++m) {
    if (m < m_lo || m >= m_hi) continue;
    const int t = t0 + tx + 16 * m;
    if (t >= L) continue;
    const long orow = out_base + (long)t * P.out_mul + P.out_add;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      if (q < q_lo || q >= q_hi) continue;
      const int c4 = co + q * 4;
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float u = acc[m][q * 4 + e];
        if (c4 + e < P.Cout) {
          u += P.bias[c4 + e];
          if (P.cond) u += P.cond[(long)b * P.cond_ld + c4 + e];
        }
        v[e] = u;
      }
      int nout = 4, oc = c4;
      if (gate) {
        v[0] = tanhf(v[0]) * (1.f / (1.f + expf(-v[1])));
        v[1] = tanhf(v[2]) * (1.f / (1.f + expf(-v[3])));
        nout = 2;
        oc = c4 >> 1;
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (e < nout) {
          float u = v[e];
          if (P.epi & EPI_RELU) u = fmaxf(u, 0.f);
          if (P.epi & EPI_TANH) u = tanhf(u);
          v[e] = u * P.alpha;
        }
      }
      float* yrow = P.y + orow * (long)P.ldy + P.yoff + oc;
      const float* rrow = P.res ? (P.res + orow * (long)P.ldr + P.roff + oc) : nullptr;
      if (aligned && !gate && (oc + 4) <= climit) {
        float4 o = make_float4(v[0], v[1], v[2], v[3]);
        if (rrow) {
          const float4 r = *reinterpret_cast<const float4*>(rrow);
          o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
        }
        *reinterpret_cast<float4*>(yrow) = o;
      } else {
        for (int e = 0; e < nout; ++e)
          if (oc + e < climit) yrow[e] = v[e] + (rrow ? rrow[e] : 0.f);
      }
      if (P.p_hi) {
        for (int e = 0; e < nout; ++e) {
          if (oc + e < climit) {
            float u = v[e] + (rrow ? rrow[e] : 0.f);
            u = u > 0.f ? u : u * P.pl_slope;
            __nv_bfloat16 hb, lb, mb;
            if (P.p_mid) { split_bf16_3(u, hb, mb, lb); P.p_mid[orow * (long)P.ldp + oc + e] = mb; }
            else split_bf16(u, hb, lb);
            P.p_hi[orow * (long)P.ldp + oc + e] = hb;
            P.p_lo[orow * (long)P.ldp + oc + e] = lb;
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Per-utterance conditioning: g = emb_g[sid] (models.py:1681); out[b][r] = W[r] . g + bias[r] for the
// stacked rows of spk_emb_linear (attentions.py:53), dp.cond (models.py:60) and every WN cond_layer
// (modules.py:151-152).
// ------------------------------------------------------------------------------------------------
__global__ void cond_kernel(const float* __restrict__ emb_g, const int* __restrict__ sid, const float* __restrict__ W,
                            const float* __restrict__ bias, float* __restrict__ out, int G, int R, int n_speakers) {
  PDL_LAUNCH();
  PDL_WAIT();
  extern __shared__ float gs[];
  const int b = blockIdx.y;
  int s = sid[b];
  s = s < 0 ? 0 : (s >= n_speakers ? n_speakers - 1 : s);      // memory-safety net for the *_dev entry points only: the host path rejects out-of-range ids
  for (int i = threadIdx.x; i < G; i += blockDim.x) gs[i] = emb_g[(long)s * G + i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + warp;
  if (r >= R) return;
  float a = 0.f;
  for (int i = lane; i < G; i += 32) a = fmaf(W[(long)r * G + i], gs[i], a);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (lane == 0) out[(long)b * R + r] = a + bias[r];
}

// Embedding * sqrt(H) (models.py:318), optional per-utterance vector (cond_layer_idx == 0).
__global__ void embed_kernel(const int* __restrict__ ids, const float* __restrict__ emb, float* __restrict__ x,
                             const int* __restrict__ lens, const int* __restrict__ offs, int H, float scale,
                             int n_vocab, const float* __restrict__ vec, int vec_ld, __nv_bfloat16* __restrict__ p_hi,
                             __nv_bfloat16* __restrict__ p_lo, __nv_bfloat16* __restrict__ p_mid) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y;
  const int t = blockIdx.x;
  if (t >= lens[b]) return;
  const long row = offs[b] + t;
  int id = ids[row];
  id = id < 0 ? 0 : (id >= n_vocab ? n_vocab - 1 : id);
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    float v = emb[(long)id * H + c] * scale;
    if (vec) v += vec[(long)b * vec_ld + c];
    x[row * H + c] = v;
    if (p_hi) {
      __nv_bfloat16 hb, lb, mb;
      if (p_mid) { split_bf16_3(v, hb, mb, lb); p_mid[row * H + c] = mb; }
      else split_bf16(v, hb, lb);
      p_hi[row * H + c] = hb;
      p_lo[row * H + c] = lb;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// out = LayerNorm_C(a + b) * gamma + beta (+ c) (+ vec[b])     (modules.py:29-32; attentions.py:59,63,
// spk add :52-56; vits2 residual models.py:377).  One warp per row, C <= 256, C % 32 == 0.
// ------------------------------------------------------------------------------------------------
__global__ void add_ln_kernel(const float* __restrict__ a, const float* __restrict__ bsrc, const float* __restrict__ gamma,
                              const float* __restrict__ beta, const float* __restrict__ cadd, const float* __restrict__ vec,
                              int vec_ld, float* __restrict__ out, const int* __restrict__ lens, const int* __restrict__ offs, int C,
                              __nv_bfloat16* __restrict__ p_hi = nullptr, __nv_bfloat16* __restrict__ p_lo = nullptr,
                              __nv_bfloat16* __restrict__ p_mid = nullptr) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * (blockDim.x >> 5) + warp;
  if (t >= lens[b]) return;
  const long row = offs[b] + t;
  const int per = C >> 5;
  float v[8];
  float s = 0.f;
  for (int i = 0; i < per; ++i) {
    const int c = lane + 32 * i;
    float u = a[row * C + c];
    if (bsrc) u += bsrc[row * C + c];
    v[i] = u;
    s += u;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  float q = 0.f;
  for (int i = 0; i < per; ++i) {
    const float d = v[i] - mean;
    q += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)C + 1e-5f);
  for (int i = 0; i < per; ++i) {
    const int c = lane + 32 * i;
    float u = (v[i] - mean) * rstd * gamma[c] + beta[c];
    if (cadd) u += cadd[row * C + c];
    if (vec) u += vec[(long)b * vec_ld + c];
    out[row * C + c] = u;
    if (p_hi) {
      __nv_bfloat16 hb, lb, mb;
      if (p_mid) { split_bf16_3(u, hb, mb, lb); p_mid[row * C + c] = mb; }
      else split_bf16(u, hb, lb);
      p_hi[row * C + c] = hb;
      p_lo[row * C + c] = lb;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Windowed relative-position multi-head self-attention (attentions.py:165-196).  The reference's
// pad/reshape skew tricks (:216-260) reduce to: score[i,j] = q_i.k_j/sqrt(dk) + [|j-i|<=W] q_i.Ek[j-i+W]/sqrt(dk),
// out_i = sum_j p_ij (v_j + [|j-i|<=W] Ev[j-i+W]).  Keys >= len are skipped: the reference fills them
// with -1e4 before the softmax (:183), whose exp underflows to exactly 0 in fp32.
// Online softmax over key tiles of 32; 4 warps x 4 query rows per CTA.
// ------------------------------------------------------------------------------------------------
constexpr int AT_KT = 32, AT_THREADS = 256;              // 8 warps; R query rows per warp -> 8*R rows per CTA
constexpr int AT_NS = 4;                                   // K/V tile ring depth (tiles are latency-, not bandwidth-bound)

constexpr int attn_smem_floats(int dk, int nrel, int R) {
  return 2 * AT_NS * AT_KT * (dk + 4) + 8 * R * (dk + 4) + 2 * nrel * (dk + 4) + 8 * R * nrel + 8 * R * AT_KT;
}

// R = 1: lowest latency (batch 1, short utterances).  R = 4: every K/V shared-memory read is reused by four query
// rows (register blocking) -- 2.5x fewer LDS per FLOP, for batched / long utterances where attention is throughput bound.
template <int DPL, int R>  // dk = 32*DPL
__global__ void __launch_bounds__(AT_THREADS)
attn_kernel(const float* __restrict__ qkv, int ld, float* __restrict__ out, int ldo, const float* __restrict__ relk,
            const float* __restrict__ relv, int n_heads, int window, const int* __restrict__ lens,
            const int* __restrict__ offs, __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo,
            __nv_bfloat16* __restrict__ p_mid) {
  PDL_LAUNCH();
  PDL_WAIT();
  constexpr int DK = 32 * DPL;
  constexpr int KS = DK + 4;              // row pitch: 16B aligned (cp.async / LDS.128), conflict-free for both access patterns
  constexpr int QT = 8 * R;
  const int b = blockIdx.z, head = blockIdx.y;
  const int len = lens[b];
  const int q0 = blockIdx.x * QT;
  if (q0 >= len) return;
  const long base = offs[b];
  const int HT = n_heads * DK;
  const int nrel = 2 * window + 1;

  extern __shared__ __align__(16) float sm[];
  float* KV = sm;                                  // [NS stages][K | V][KT][KS]
  float* Qs = KV + 2 * AT_NS * AT_KT * KS;         // [QT][KS]
  float* Rk = Qs + QT * KS;                        // [nrel][KS]
  float* Rv = Rk + nrel * KS;                      // [nrel][KS]
  float* QE = Rv + nrel * KS;                      // [QT][nrel]
  float* Ps = QE + QT * nrel;                      // [QT][KT]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ntiles = (len + AT_KT - 1) / AT_KT;

  auto issue_tile = [&](int kt) {
    float* kd = KV + (kt % AT_NS) * 2 * AT_KT * KS;
    float* vd = kd + AT_KT * KS;
    const int k0 = kt * AT_KT;
    for (int i = tid; i < AT_KT * (DK / 4); i += AT_THREADS) {
      const int r = i / (DK / 4), d4 = (i - r * (DK / 4)) * 4;
      const int t = k0 + r;
      const bool ok = t < len;
      const float* rowp = qkv + (base + (ok ? t : 0)) * (long)ld + head * DK + d4;
      cp_async16(kd + r * KS + d4, rowp + HT, ok ? 16 : 0);
      cp_async16(vd + r * KS + d4, rowp + 2 * HT, ok ? 16 : 0);
    }
  };
#pragma unroll
  for (int i = 0; i < AT_NS - 1; ++i) {
    if (i < ntiles) issue_tile(i);
    cp_async_commit();
  }

  // Q rows (pre-scaled by 1/sqrt(dk) as attentions.py:171 does) and both relative-position tables into shared memory
  for (int i = tid; i < QT * (DK / 4); i += AT_THREADS) {
    const int r = i / (DK / 4), d4 = (i - r * (DK / 4)) * 4;
    const int t = q0 + r;
    float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < len) q = *reinterpret_cast<const float4*>(qkv + (base + t) * (long)ld + head * DK + d4);
    const float sc = sqrtf((float)DK);
    q.x /= sc; q.y /= sc; q.z /= sc; q.w /= sc;
    *reinterpret_cast<float4*>(Qs + r * KS + d4) = q;
  }
  for (int i = tid; i < nrel * (DK / 4); i += AT_THREADS) {
    const int r = i / (DK / 4), d4 = (i - r * (DK / 4)) * 4;
    *reinterpret_cast<float4*>(Rk + r * KS + d4) = *reinterpret_cast<const float4*>(relk + r * DK + d4);
    *reinterpret_cast<float4*>(Rv + r * KS + d4) = *reinterpret_cast<const float4*>(relv + r * DK + d4);
  }
  __syncthreads();
  // q . Ek for the 2W+1 relative offsets: one thread per (row, offset)
  for (int i = tid; i < QT * nrel; i += AT_THREADS) {
    const int r = i / nrel, m = i - r * nrel;
    float a = 0.f;
#pragma unroll 4
    for (int d4 = 0; d4 < DK; d4 += 4) {
      const float4 q = *reinterpret_cast<const float4*>(Qs + r * KS + d4);
      const float4 e = *reinterpret_cast<const float4*>(Rk + m * KS + d4);
      a = fmaf(q.x, e.x, a); a = fmaf(q.y, e.y, a); a = fmaf(q.z, e.z, a); a = fmaf(q.w, e.w, a);
    }
    QE[i] = a;
  }
  timeline_stamp(-11);

  float mrun[R], lrun[R], acc[R][DPL];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    mrun[r] = -INFINITY;
    lrun[r] = 0.f;
#pragma unroll
    for (int e = 0; e < DPL; ++e) acc[r][e] = 0.f;
  }
  const int row0 = warp * R;                       // first local query row of this warp

  for (int kt = 0; kt < ntiles; ++kt) {
    const int k0 = kt * AT_KT;
    if (kt + AT_NS - 1 < ntiles) issue_tile(kt + AT_NS - 1);   // its ring slot was consumed in iteration kt-1 (barrier below)
    cp_async_commit();
    cp_async_wait<AT_NS - 1>();
    __syncthreads();                             // tile kt landed; QE visible (first iteration)
    if (kt == 0) timeline_stamp(-12);
    const float* Ks = KV + (kt % AT_NS) * 2 * AT_KT * KS;
    const float* Vs = Ks + AT_KT * KS;
    const int key = k0 + lane;
    const bool kvalid = key < len;
    float s0[R], s1[R], s2[R], s3[R];              // four independent chains per row (the 4-cycle FMA latency is the limiter)
#pragma unroll
    for (int r = 0; r < R; ++r) s0[r] = s1[r] = s2[r] = s3[r] = 0.f;
#pragma unroll
    for (int d4 = 0; d4 < DK; d4 += 4) {
      const float4 kd = *reinterpret_cast<const float4*>(Ks + lane * KS + d4);
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float4 qd = *reinterpret_cast<const float4*>(Qs + (row0 + r) * KS + d4);
        s0[r] = fmaf(qd.x, kd.x, s0[r]); s1[r] = fmaf(qd.y, kd.y, s1[r]);
        s2[r] = fmaf(qd.z, kd.z, s2[r]); s3[r] = fmaf(qd.w, kd.w, s3[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int qi = q0 + row0 + r;
      float s = (s0[r] + s1[r]) + (s2[r] + s3[r]);
      const int rel = key - qi + window;
      if (rel >= 0 && rel < nrel) s += QE[(row0 + r) * nrel + rel];
      if (!kvalid) s = -INFINITY;
      float mx = s;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float mnew = fmaxf(mrun[r], mx);
      const float corr = expf(mrun[r] - mnew);
      const float p = kvalid ? expf(s - mnew) : 0.f;
      float ps = p;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, o);
      lrun[r] = lrun[r] * corr + ps;
      mrun[r] = mnew;
#pragma unroll
      for (int e = 0; e < DPL; ++e) acc[r][e] *= corr;
      Ps[(row0 + r) * AT_KT + lane] = p;
    }
    __syncwarp();
    const int kmax = min(AT_KT, len - k0);
    if (kmax == AT_KT) {
      float a2[R][DPL];
#pragma unroll
      for (int r = 0; r < R; ++r)
#pragma unroll
        for (int e = 0; e < DPL; ++e) a2[r][e] = 0.f;
#pragma unroll
      for (int kk = 0; kk < AT_KT; kk += 2) {            // fully unrolled, two accumulator sets
        float v0[DPL], v1[DPL];
#pragma unroll
        for (int e = 0; e < DPL; ++e) { v0[e] = Vs[kk * KS + lane + 32 * e]; v1[e] = Vs[(kk + 1) * KS + lane + 32 * e]; }
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const float p0 = Ps[(row0 + r) * AT_KT + kk], p1 = Ps[(row0 + r) * AT_KT + kk + 1];
#pragma unroll
          for (int e = 0; e < DPL; ++e) {
            acc[r][e] = fmaf(p0, v0[e], acc[r][e]);
            a2[r][e] = fmaf(p1, v1[e], a2[r][e]);
          }
        }
      }
#pragma unroll
      for (int r = 0; r < R; ++r)
#pragma unroll
        for (int e = 0; e < DPL; ++e) acc[r][e] += a2[r][e];
    } else {
      for (int kk = 0; kk < kmax; ++kk) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const float pk = Ps[(row0 + r) * AT_KT + kk];
#pragma unroll
          for (int e = 0; e < DPL; ++e) acc[r][e] = fmaf(pk, Vs[kk * KS + lane + 32 * e], acc[r][e]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int qi = q0 + row0 + r;
      for (int m = 0; m < nrel; ++m) {
        const int kk = qi + m - window - k0;
        if (kk >= 0 && kk < kmax) {
          const float pk = Ps[(row0 + r) * AT_KT + kk];
#pragma unroll
          for (int e = 0; e < DPL; ++e) acc[r][e] = fmaf(pk, Rv[m * KS + lane + 32 * e], acc[r][e]);
        }
      }
    }
    __syncthreads();   // tile buffer and Ps fully consumed before the next prefetch overwrites them
  }
  timeline_stamp(-13);
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int qi = q0 + row0 + r;
    if (qi < len) {
      const float inv = 1.f / lrun[r];
#pragma unroll
      for (int e = 0; e < DPL; ++e) {
        const float o = acc[r][e] * inv;
        const long idx = (base + qi) * (long)ldo + head * DK + lane + 32 * e;
        out[idx] = o;
        if (p_hi) {
          __nv_bfloat16 hb, lb, mb;
          if (p_mid) { split_bf16_3(o, hb, mb, lb); p_mid[idx] = mb; }
          else split_bf16(o, hb, lb);
          p_hi[idx] = hb;
          p_lo[idx] = lb;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Split-KV variant of the attention for single short utterances (latency bound: a warp of attn_kernel walks all key
// tiles of its row serially, ~1.8 us per tile).  One CTA = 4 query rows of one head, 16 warps; all K/V tiles of the utterance
// (<= ATS_MAXT) are resident in shared memory; warp w handles row w%4 and the key tiles {w/4, w/4+4}; the four
// partial (max, sum, accumulator) states of a row are merged in segment order at the end.
// ------------------------------------------------------------------------------------------------
constexpr int ATS_ROWS = 4, ATS_SEG = 4, ATS_MAXT = 8, ATS_WARPS = ATS_ROWS * ATS_SEG, ATS_THREADS = 32 * ATS_WARPS;
constexpr int ATS_SMEM_MAX = 227 * 1024;          // dynamic shared memory the split-KV kernel is allowed (sm_90 maximum)
constexpr int attn_split_smem_floats(int dk, int nrel, int ntiles) {
  return 2 * ntiles * AT_KT * (dk + 4) + ATS_ROWS * (dk + 4) + 2 * nrel * (dk + 4) + ATS_ROWS * nrel + ATS_WARPS * AT_KT + ATS_WARPS * (4 + dk);
}

template <int DPL>  // dk = 32*DPL
__global__ void __launch_bounds__(ATS_THREADS)
attn_split_kernel(const float* __restrict__ qkv, int ld, float* __restrict__ out, int ldo, const float* __restrict__ relk,
                  const float* __restrict__ relv, int n_heads, int window, int max_tiles, const int* __restrict__ lens,
                  const int* __restrict__ offs, __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo,
                  __nv_bfloat16* __restrict__ p_mid) {
  PDL_LAUNCH();
  constexpr int DK = 32 * DPL;
  constexpr int KS = DK + 4;
  const int b = blockIdx.z, head = blockIdx.y;
  const int nrel = 2 * window + 1;
  extern __shared__ __align__(16) float sm[];
  float* KV = sm;                                   // [max_tiles][K | V][KT][KS]
  float* Qs = KV + 2 * max_tiles * AT_KT * KS;      // [ROWS][KS]
  float* Rk = Qs + ATS_ROWS * KS;                   // [nrel][KS]
  float* Rv = Rk + nrel * KS;                       // [nrel][KS]
  float* QE = Rv + nrel * KS;                       // [2][nrel]
  float* Ps = QE + ATS_ROWS * nrel;                 // [8 warps][KT]
  float* Mg = Ps + ATS_WARPS * AT_KT;               // [warps][4 + DK]  (m, l, -, -, acc[DK])
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // the relative-position tables are constants: staged before the dependency wait
  for (int i = tid; i < nrel * (DK / 4); i += ATS_THREADS) {
    const int r = i / (DK / 4), d4 = (i - r * (DK / 4)) * 4;
    *reinterpret_cast<float4*>(Rk + r * KS + d4) = *reinterpret_cast<const float4*>(relk + r * DK + d4);
    *reinterpret_cast<float4*>(Rv + r * KS + d4) = *reinterpret_cast<const float4*>(relv + r * DK + d4);
  }
  PDL_WAIT();
  const int len = lens[b];
  const int q0 = blockIdx.x * ATS_ROWS;
  if (q0 >= len) return;
  const long base = offs[b];
  const int HT = n_heads * DK;
  const int ntiles = (len + AT_KT - 1) / AT_KT;     // <= max_tiles (host guarantees)

  auto issue_tile = [&](int kt) {
    float* kd = KV + kt * 2 * AT_KT * KS;
    float* vd = kd + AT_KT * KS;
    const int k0 = kt * AT_KT;
    for (int i = tid; i < AT_KT * (DK / 4); i += ATS_THREADS) {
      const int r = i / (DK / 4), d4 = (i - r * (DK / 4)) * 4;
      const int t = k0 + r;
      const bool ok = t < len;
      const float* rowp = qkv + (base + (ok ? t : 0)) * (long)ld + head * DK + d4;
      cp_async16(kd + r * KS + d4, rowp + HT, ok ? 16 : 0);
      cp_async16(vd + r * KS + d4, rowp + 2 * HT, ok ? 16 : 0);
    }
  };
  // two commit groups: the tiles of the first round (0..3) and of the second (4..7)
  for (int kt = 0; kt < min(ntiles, ATS_SEG); ++kt) issue_tile(kt);
  cp_async_commit();
  for (int kt = ATS_SEG; kt < ntiles; ++kt) issue_tile(kt);
  cp_async_commit();

  for (int i = tid; i < ATS_ROWS * (DK / 4); i += ATS_THREADS) {
    const int r = i / (DK / 4), d4 = (i - r * (DK / 4)) * 4;
    const int t = q0 + r;
    float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < len) q = *reinterpret_cast<const float4*>(qkv + (base + t) * (long)ld + head * DK + d4);
    const float sc = sqrtf((float)DK);
    q.x /= sc; q.y /= sc; q.z /= sc; q.w /= sc;
    *reinterpret_cast<float4*>(Qs + r * KS + d4) = q;
  }
  __syncthreads();
  for (int i = tid; i < ATS_ROWS * nrel; i += ATS_THREADS) {
    const int r = i / nrel, m = i - r * nrel;
    float a = 0.f;
#pragma unroll 4
    for (int d4 = 0; d4 < DK; d4 += 4) {
      const float4 q = *reinterpret_cast<const float4*>(Qs + r * KS + d4);
      const float4 e = *reinterpret_cast<const float4*>(Rk + m * KS + d4);
      a = fmaf(q.x, e.x, a); a = fmaf(q.y, e.y, a); a = fmaf(q.z, e.z, a); a = fmaf(q.w, e.w, a);
    }
    QE[i] = a;
  }

  const int row = warp % ATS_ROWS, seg = warp / ATS_ROWS;
  const int qi = q0 + row;
  float mrun = -INFINITY, lrun = 0.f, acc[DPL];
#pragma unroll
  for (int e = 0; e < DPL; ++e) acc[e] = 0.f;
  float* Pw = Ps + warp * AT_KT;

#pragma unroll 1
  for (int round = 0; round < 2; ++round) {
    if (round == 0) cp_async_wait<1>(); else cp_async_wait<0>();
    __syncthreads();                               // this round's tiles (and QE) visible to every warp
    const int kt = seg + round * ATS_SEG;
    if (kt >= ntiles) continue;                    // (uniform per warp; the barriers above are outside the branch)
    const int k0 = kt * AT_KT;
    const float* Ks = KV + kt * 2 * AT_KT * KS;
    const float* Vs = Ks + AT_KT * KS;
    const int key = k0 + lane;
    const bool kvalid = key < len;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
    for (int d4 = 0; d4 < DK; d4 += 4) {
      const float4 kd = *reinterpret_cast<const float4*>(Ks + lane * KS + d4);
      const float4 qd = *reinterpret_cast<const float4*>(Qs + row * KS + d4);
      s0 = fmaf(qd.x, kd.x, s0); s1 = fmaf(qd.y, kd.y, s1); s2 = fmaf(qd.z, kd.z, s2); s3 = fmaf(qd.w, kd.w, s3);
    }
    float sc = (s0 + s1) + (s2 + s3);
    const int rel = key - qi + window;
    if (rel >= 0 && rel < nrel) sc += QE[row * nrel + rel];
    if (!kvalid) sc = -INFINITY;
    float mx = sc;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float mnew = fmaxf(mrun, mx);
    const float corr = expf(mrun - mnew);
    const float p = kvalid ? expf(sc - mnew) : 0.f;
    float ps = p;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, o);
    lrun = lrun * corr + ps;
    mrun = mnew;
#pragma unroll
    for (int e = 0; e < DPL; ++e) acc[e] *= corr;
    Pw[lane] = p;
    __syncwarp();
    const int kmax = min(AT_KT, len - k0);
    float a2[DPL];
#pragma unroll
    for (int e = 0; e < DPL; ++e) a2[e] = 0.f;
    int kk = 0;
    for (; kk + 1 < kmax; kk += 2) {
      const float p0 = Pw[kk], p1 = Pw[kk + 1];
#pragma unroll
      for (int e = 0; e < DPL; ++e) {
        acc[e] = fmaf(p0, Vs[kk * KS + lane + 32 * e], acc[e]);
        a2[e] = fmaf(p1, Vs[(kk + 1) * KS + lane + 32 * e], a2[e]);
      }
    }
    if (kk < kmax) {
      const float p0 = Pw[kk];
#pragma unroll
      for (int e = 0; e < DPL; ++e) acc[e] = fmaf(p0, Vs[kk * KS + lane + 32 * e], acc[e]);
    }
#pragma unroll
    for (int e = 0; e < DPL; ++e) acc[e] += a2[e];
    for (int m = 0; m < nrel; ++m) {
      const int kr = qi + m - window - k0;
      if (kr >= 0 && kr < kmax) {
        const float pk = Pw[kr];
#pragma unroll
        for (int e = 0; e < DPL; ++e) acc[e] = fmaf(pk, Rv[m * KS + lane + 32 * e], acc[e]);
      }
    }
    __syncwarp();                                  // Pw is rewritten in the next round
  }
  // merge the four segments of each row (segment order => deterministic)
  float* mg = Mg + warp * (4 + DK);
  if (lane == 0) { mg[0] = mrun; mg[1] = lrun; }
#pragma unroll
  for (int e = 0; e < DPL; ++e) mg[4 + lane + 32 * e] = acc[e];
  __syncthreads();
  if (seg == 0 && qi < len) {
    float mstar = -INFINITY;
#pragma unroll
    for (int g = 0; g < ATS_SEG; ++g) mstar = fmaxf(mstar, Mg[(row + ATS_ROWS * g) * (4 + DK)]);
    float l = 0.f, o[DPL];
#pragma unroll
    for (int e = 0; e < DPL; ++e) o[e] = 0.f;
#pragma unroll
    for (int g = 0; g < ATS_SEG; ++g) {
      const float* pg = Mg + (row + ATS_ROWS * g) * (4 + DK);
      const float w = expf(pg[0] - mstar);         // exp(-inf) = 0 for a segment that had no tile
      l = fmaf(pg[1], w, l);
#pragma unroll
      for (int e = 0; e < DPL; ++e) o[e] = fmaf(pg[4 + lane + 32 * e], w, o[e]);
    }
    const float inv = 1.f / l;
#pragma unroll
    for (int e = 0; e < DPL; ++e) {
      const float v = o[e] * inv;
      const long idx = (base + qi) * (long)ldo + head * DK + lane + 32 * e;
      out[idx] = v;
      if (p_hi) {
        __nv_bfloat16 hb, lb, mb;
        if (p_mid) { split_bf16_3(v, hb, mb, lb); p_mid[idx] = mb; }
        else split_bf16(v, hb, lb);
        p_hi[idx] = hb;
        p_lo[idx] = lb;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// One DDSConv layer (modules.py:96-108): depthwise dilated conv k -> LN -> GELU(erf) -> 1x1 -> LN ->
// GELU -> + x.  One CTA = 8 positions x all C channels (C == blockDim.x <= 256).
// ------------------------------------------------------------------------------------------------
constexpr int DDS_TT = 4;      // positions per CTA
constexpr int DDS_CH = 32;     // 1x1 weight rows (input channels) per cp.async chunk
constexpr int DDS_NS = 4;      // chunk ring depth

struct DdsP {
  const float* x;
  // ConvFlow front fused into the first layer (modules.py:366-367 + DDSConv's `x = x + g`, :97-98): when x0 is set the
  // layer's input is h[t][c] = pre_w[c] * x0[t] + pre_b[c] + cond[t][c] instead of x (same op order as the separate kernel)
  const float* x0;
  const float* pre_w;
  const float* pre_b;
  const float* cond;
  float* y;
  const float *sep_w, *sep_b, *ln1g, *ln1b, *pw_w, *pw_b, *ln2g, *ln2b;
  int C, k, dil, ldw;
};

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }

template <int TT>
__device__ __forceinline__ void block_ln_stats(float (&v)[TT], float* red, int C, float (&mean)[TT], float (&rstd)[TT]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  float s[TT];
#pragma unroll
  for (int i = 0; i < TT; ++i) {
    s[i] = v[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s[i] += __shfl_xor_sync(0xffffffffu, s[i], o);
  }
  __syncthreads();
  if (lane == 0)
#pragma unroll
    for (int i = 0; i < TT; ++i) red[warp * TT + i] = s[i];
  __syncthreads();
#pragma unroll
  for (int i = 0; i < TT; ++i) {
    float t = 0.f;
    for (int w = 0; w < nw; ++w) t += red[w * TT + i];
    mean[i] = t / (float)C;
  }
#pragma unroll
  for (int i = 0; i < TT; ++i) {
    const float d = v[i] - mean[i];
    s[i] = d * d;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s[i] += __shfl_xor_sync(0xffffffffu, s[i], o);
  }
  __syncthreads();
  if (lane == 0)
#pragma unroll
    for (int i = 0; i < TT; ++i) red[warp * TT + i] = s[i];
  __syncthreads();
#pragma unroll
  for (int i = 0; i < TT; ++i) {
    float t = 0.f;
    for (int w = 0; w < nw; ++w) t += red[w * TT + i];
    rstd[i] = rsqrtf(t / (float)C + 1e-5f);
  }
}

// One CTA = TT positions x all C channels (TT = TT for single utterances: more CTAs; TTB for batches: every CTA streams
// the whole 1x1 weight matrix, so more positions per CTA means less L2 traffic and more FFMAs per shared-memory read;
// the arithmetic per position is the same in both) (thread c owns channel c).  The 1x1 weight matrix streams through a
// 3-deep cp.async ring of 32-row chunks; the first chunks are in flight while the depthwise conv and LN run.
template <int TT>
__global__ void __launch_bounds__(256)
dds_layer_kernel(const DdsP P, const int* __restrict__ lens, const int* __restrict__ offs) {
  PDL_LAUNCH();
  // token lengths/offsets are uploaded by host copies ordered before the graph, never produced by a predecessor kernel:
  // they (and the immutable weights) may be touched before PDL_WAIT
  const int b = blockIdx.y;
  const int len = lens[b];
  const int t0 = blockIdx.x * TT;
  if (t0 >= len) return;
  const long base = offs[b];
  const int C = P.C, c = threadIdx.x;
  extern __shared__ __align__(16) float dsm[];
  float* Wr = dsm;                                   // [NS][CH][C]
  float* ys = Wr + DDS_NS * DDS_CH * C;              // [C][TT]
  float* red = ys + C * TT;                      // [8][TT]
  const int nch = C / DDS_CH;
  __shared__ uint64_t wfull[DDS_NS];
  if (c == 0) {
    for (int i = 0; i < DDS_NS; ++i) mbar_init(&wfull[i], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // one 32-row chunk of the 1x1 weight matrix = one contiguous bulk copy (ldw == C), issued by a single thread
  auto issue_chunk = [&](int ch) {
    if (c == 0) {
      const int slot = ch % DDS_NS;
      const uint32_t bytes = (uint32_t)(DDS_CH * C * sizeof(float));
      mbar_expect_tx(&wfull[slot], bytes);
      bulk_copy_g2s(Wr + slot * DDS_CH * C, P.pw_w + (long)ch * DDS_CH * P.ldw, bytes, &wfull[slot]);
    }
  };
#pragma unroll
  for (int i = 0; i < DDS_NS - 1; ++i)
    if (i < nch) issue_chunk(i);
  PDL_WAIT();                                        // P.x comes from the previous kernel

  float v[TT], mean[TT], rstd[TT];
  const int half = (P.k - 1) / 2;
  const float fpw = P.x0 ? P.pre_w[c] : 0.f, fpb = P.x0 ? P.pre_b[c] : 0.f;
  auto ld_x = [&](int t) -> float {
    const long row = base + t;
    if (P.x0) return fmaf(fpw, P.x0[row], fpb) + P.cond[row * (long)C + c];
    return P.x[row * (long)C + c];
  };
#pragma unroll
  for (int i = 0; i < TT; ++i) {
    float a = P.sep_b[c];
    for (int j = 0; j < P.k; ++j) {
      const int t = t0 + i + (j - half) * P.dil;
      if (t >= 0 && t < len) a = fmaf(P.sep_w[j * C + c], ld_x(t), a);
    }
    v[i] = a;
  }
  timeline_stamp(-1);
  block_ln_stats<TT>(v, red, C, mean, rstd);
  timeline_stamp(-2);
  {
    const float g = P.ln1g[c], be = P.ln1b[c];
#pragma unroll
    for (int i = 0; i < TT; i += 4) {
      float4 o;
      o.x = gelu_erf((v[i] - mean[i]) * rstd[i] * g + be);
      o.y = gelu_erf((v[i + 1] - mean[i + 1]) * rstd[i + 1] * g + be);
      o.z = gelu_erf((v[i + 2] - mean[i + 2]) * rstd[i + 2] * g + be);
      o.w = gelu_erf((v[i + 3] - mean[i + 3]) * rstd[i + 3] * g + be);
      *reinterpret_cast<float4*>(ys + c * TT + i) = o;
    }
  }
  {
    const float bias = P.pw_b[c];
#pragma unroll
    for (int i = 0; i < TT; ++i) v[i] = bias;
  }
  for (int ch = 0; ch < nch; ++ch) {
    __syncthreads();                                 // ys visible (first iteration); slot (ch-1)%NS has been consumed
    if (ch + DDS_NS - 1 < nch) issue_chunk(ch + DDS_NS - 1);
    mbar_wait(&wfull[ch % DDS_NS], (ch / DDS_NS) & 1);   // chunk ch landed
    const float* wr = Wr + (ch % DDS_NS) * DDS_CH * C + c;
    const float* yy = ys + ch * DDS_CH * TT;
#pragma unroll 8
    for (int ci = 0; ci < DDS_CH; ++ci) {
      const float w = wr[ci * C];
#pragma unroll
      for (int i = 0; i < TT; i += 4) {
        const float4 y0 = *reinterpret_cast<const float4*>(yy + ci * TT + i);
        v[i] = fmaf(w, y0.x, v[i]); v[i + 1] = fmaf(w, y0.y, v[i + 1]); v[i + 2] = fmaf(w, y0.z, v[i + 2]); v[i + 3] = fmaf(w, y0.w, v[i + 3]);
      }
    }
  }
  timeline_stamp(-3);
  block_ln_stats<TT>(v, red, C, mean, rstd);
  timeline_stamp(-4);
  {
    const float g = P.ln2g[c], be = P.ln2b[c];
#pragma unroll
    for (int i = 0; i < TT; ++i) {
      const int t = t0 + i;
      if (t < len) {
        const long idx = (base + t) * (long)C + c;
        P.y[idx] = ld_x(t) + gelu_erf((v[i] - mean[i]) * rstd[i] * g + be);
      }
    }
  }
}

// ConvFlow front (modules.py:366-367 + DDSConv's `x = x + g`, :97-98): h = pre_w * x0 + pre_b + cond.
__global__ void cf_pre_kernel(const float* __restrict__ x0, const float* __restrict__ pre_w, const float* __restrict__ pre_b,
                              const float* __restrict__ cond, float* __restrict__ h, const int* __restrict__ lens,
                              const int* __restrict__ offs, int C) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= lens[b]) return;
  const long row = offs[b] + t;
  const float xv = x0[row];
  for (int c = threadIdx.x; c < C; c += blockDim.x) h[row * C + c] = fmaf(pre_w[c], xv, pre_b[c]) + cond[row * C + c];
}

// z = eps * noise_scale_w (models.py:96); eps either supplied ([B][2][ld]) or Philox.
__device__ __forceinline__ void philox4x32(uint32_t (&ctr)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr[0]), lo0 = 0xD2511F53u * ctr[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr[2]), lo1 = 0xCD9E8D57u * ctr[2];
    const uint32_t n0 = hi1 ^ ctr[1] ^ k0, n1 = lo1, n2 = hi0 ^ ctr[3] ^ k1, n3 = lo0;
    ctr[0] = n0; ctr[1] = n1; ctr[2] = n2; ctr[3] = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}
__device__ __forceinline__ float philox_normal(uint64_t seed, uint32_t stream, uint32_t a, uint32_t bidx) {
  uint32_t ctr[4] = {a, bidx, stream, 0x5eedu};
  philox4x32(ctr, (uint32_t)seed, (uint32_t)(seed >> 32));
  const float u1 = ((float)(ctr[0] >> 8) + 0.5f) * (1.f / 16777216.f);
  const float u2 = ((float)(ctr[1] >> 8) + 0.5f) * (1.f / 16777216.f);
  return sqrtf(-2.f * logf(u1)) * cospif(2.f * u2);
}

// Per-call scalars live in a small device block so that captured CUDA graphs stay valid across calls:
//   prm[0] noise_scale, prm[1] length_scale, prm[2] noise_scale_w, prm[4..5] Philox seed (lo, hi as raw bits).
__device__ __forceinline__ uint64_t prm_seed(const float* prm) {
  return (uint64_t)__float_as_uint(prm[4]) | ((uint64_t)__float_as_uint(prm[5]) << 32);
}

__global__ void dp_noise_kernel(const float* __restrict__ eps, int eps_ld, const float* __restrict__ prm, float* __restrict__ za,
                                float* __restrict__ zb, const int* __restrict__ lens, const int* __restrict__ offs) {
  PDL_LAUNCH();
  PDL_WAIT();
  const uint64_t seed = prm_seed(prm);
  const float scale = prm[2];
  const int b = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= lens[b]) return;
  const long row = offs[b] + t;
  float e0, e1;
  if (eps) {
    e0 = eps[((long)b * 2 + 0) * eps_ld + t];
    e1 = eps[((long)b * 2 + 1) * eps_ld + t];
  } else {
    e0 = philox_normal(seed, 1u, (uint32_t)t, (uint32_t)(2 * b));
    e1 = philox_normal(seed, 1u, (uint32_t)t, (uint32_t)(2 * b + 1));
  }
  za[row] = e0 * scale;
  zb[row] = e1 * scale;
}

// ------------------------------------------------------------------------------------------------
// Inverse rational-quadratic spline with linear tails (transforms.py:55-193, inverse branch) applied to
// x1 given the 3*nb-1 parameters of one position (modules.py:373-385).  Op order follows the reference
// (no FMA contraction) because ceil() of the resulting duration must be bit-stable.
// ------------------------------------------------------------------------------------------------
constexpr int SPL_MAXB = 16;
// row pitch of the parameter rows: 3 * nb - 1 floats (widths, heights, interior derivatives) padded to a float4
constexpr int spline_pitch(int nb) { return (3 * nb - 1 + 3) / 4 * 4; }

__global__ void spline_inverse_kernel(const float* __restrict__ h, int ldh, float* __restrict__ x1, int nb, float bound,
                                      float sqrt_filter, const int* __restrict__ lens, const int* __restrict__ offs) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= lens[b]) return;
  const long row = offs[b] + t;
  const float x = x1[row];
  if (!(x >= -bound && x <= bound)) return;  // linear tails: identity (transforms.py:77)
  const float* hp = h + row * (long)ldh;
  float cw[SPL_MAXB + 1], ch[SPL_MAXB + 1], dv[SPL_MAXB + 1];
  const float den = sqrt_filter;  // h / math.sqrt(filter_channels)  (modules.py:373-374)
  const float coef = (float)(1.0 - 1e-3 * (double)nb);  // python evaluates (1 - min_bin_width*num_bins) in double
  for (int pass = 0; pass < 2; ++pass) {
    float* cum = pass == 0 ? cw : ch;
    float u[SPL_MAXB];
    float mx = -INFINITY;
    for (int i = 0; i < nb; ++i) {
      u[i] = __fdiv_rn(hp[pass * nb + i], den);
      mx = fmaxf(mx, u[i]);
    }
    float s = 0.f;
    for (int i = 0; i < nb; ++i) {
      u[i] = expf(__fsub_rn(u[i], mx));
      s = __fadd_rn(s, u[i]);
    }
    float run = 0.f;
    cum[0] = -bound;
    for (int i = 0; i < nb; ++i) {
      const float wi = __fadd_rn(1e-3f, __fmul_rn(coef, __fdiv_rn(u[i], s)));
      run = __fadd_rn(run, wi);
      cum[i + 1] = __fadd_rn(__fmul_rn(2.f * bound, run), -bound);
    }
    cum[nb] = bound;
  }
  const float cst = 0.5397424172369522f;  // log(exp(1 - 1e-3) - 1)  (transforms.py:73)
  for (int i = 0; i <= nb; ++i) {
    const float ud = (i == 0 || i == nb) ? cst : hp[2 * nb + i - 1];
    const float sp = ud > 20.f ? ud : log1pf(expf(ud));
    dv[i] = __fadd_rn(1e-3f, sp);
  }
  int bin = -1;
  for (int i = 0; i <= nb; ++i) {
    const float loc = (i == nb) ? __fadd_rn(ch[i], 1e-6f) : ch[i];
    bin += (x >= loc) ? 1 : 0;
  }
  bin = bin < 0 ? 0 : (bin > nb - 1 ? nb - 1 : bin);
  const float in_cw = cw[bin], in_w = __fsub_rn(cw[bin + 1], cw[bin]);
  const float in_ch = ch[bin], in_h = __fsub_rn(ch[bin + 1], ch[bin]);
  const float delta = __fdiv_rn(in_h, in_w);
  const float d0 = dv[bin], d1 = dv[bin + 1];
  const float tsum = __fsub_rn(__fadd_rn(d0, d1), __fmul_rn(2.f, delta));
  const float dx = __fsub_rn(x, in_ch);
  const float a = __fadd_rn(__fmul_rn(dx, tsum), __fmul_rn(in_h, __fsub_rn(delta, d0)));
  const float bq = __fsub_rn(__fmul_rn(in_h, d0), __fmul_rn(dx, tsum));
  const float c = __fmul_rn(-delta, dx);
  const float disc = __fsub_rn(__fmul_rn(bq, bq), __fmul_rn(__fmul_rn(4.f, a), c));
  const float root = __fdiv_rn(__fmul_rn(2.f, c), __fsub_rn(-bq, __fsqrt_rn(disc)));
  x1[row] = __fadd_rn(__fmul_rn(root, in_w), in_cw);
}

constexpr int SEQ_GAP = 8;
// ------------------------------------------------------------------------------------------------
// Durations (models.py:1689-1691; modules.py:296 for the ElementwiseAffine inverse):
//   logw = (z - m) * exp(-logs);  w = exp(logw) * length_scale;  w_ceil = ceil(w);  cum = cumsum(w_ceil)
// One CTA per utterance; y_len = max(sum, 1).  A token has at most 1e6 frames, so one 256-token pass sums to well inside
// an int, but a long utterance or batch can pass INT32_MAX frames: the running sums are 64-bit, and an utterance whose frames
// do not fit an int gets y_len -1, a batch whose frame layout does not fit gets the total offset -1 (the host refuses both).
// ------------------------------------------------------------------------------------------------
__global__ void duration_kernel(const float* __restrict__ z, const float* __restrict__ ea, int ea_ch, int ea_n, const float* __restrict__ prm,
                                int* __restrict__ wceil, int* __restrict__ cum, int* __restrict__ ylen,
                                const int* __restrict__ lens, const int* __restrict__ offs,
                                int* __restrict__ yoff, int B, volatile int* host_out, unsigned int* __restrict__ done_counter,
                                int* __restrict__ ylen_real) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.x;
  const int len = lens[b];
  const long base = offs[b];
  __shared__ int part[1024];
  __shared__ long long carry;
  const float length_scale = prm[1];
  const float m = ea[ea_ch], nlogs = -ea[ea_n + ea_ch];
  const float es = expf(nlogs);
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int t0 = 0; t0 < len; t0 += blockDim.x) {
    const int t = t0 + threadIdx.x;
    int wc = 0;
    if (t < len) {
      const float logw = __fmul_rn(__fsub_rn(z[base + t], m), es);
      const float w = __fmul_rn(expf(logw), length_scale);
      float c = ceilf(w);
      c = fminf(fmaxf(c, 0.f), 1.0e6f);
      wc = (int)c;
      wceil[base + t] = wc;
    }
    part[threadIdx.x] = wc;
    __syncthreads();
    for (int o = 1; o < blockDim.x; o <<= 1) {
      int add = threadIdx.x >= o ? part[threadIdx.x - o] : 0;
      __syncthreads();
      part[threadIdx.x] += add;
      __syncthreads();
    }
    if (t < len) cum[base + t] = (int)(carry + part[threadIdx.x]);
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry += part[threadIdx.x];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    ylen[b] = carry > (long long)INT_MAX ? -1 : (carry < 1 ? 1 : (int)carry);
    // the block that finishes last lays the utterances out at frame resolution and publishes lengths + offsets to the host
    // (what frame_offsets_kernel does as a separate launch)
    __threadfence();
    const unsigned int ticket = atomicAdd(done_counter, 1u);
    if (ticket == (unsigned int)B - 1u) {
      __threadfence();
      // prm[7] > 0: the host has already enqueued the second phase for a PREDICTED length bucket of that many frames
      // (speculative phase 2).  Its buffers, tensor maps and grids are sized for the bucket, so the device-side lengths it
      // reads are clamped to it; the host gets the true lengths, sees that the prediction was too small and repeats the
      // phase after restoring them from ylen_real (restore_lengths_kernel).
      // (an utterance refused for its length, y_len -1, runs as `cap` frames in an already enqueued second phase)
      const int cap = __float_as_int(prm[7]);
      long long o = 0, o_real = 0;
      for (int b2 = 0; b2 < B; ++b2) {
        const int yl = *((volatile int*)&ylen[b2]);
        ylen_real[b2] = yl;
        const int ylc = (cap > 0 && (yl > cap || yl < 1)) ? cap : yl;
        if (ylc != yl) ylen[b2] = ylc;
        yoff[b2] = (int)o;
        if (host_out) { host_out[1 + b2] = yl; host_out[1 + B + b2] = (int)o_real; }
        o += ylc + (b2 + 1 < B ? SEQ_GAP : 0);
        o_real += (long long)yl + (b2 + 1 < B ? SEQ_GAP : 0);
      }
      const bool too_long = o_real > (long long)INT_MAX;
      yoff[B] = too_long ? -1 : (int)o;
      if (host_out) {
        host_out[1 + 2 * B] = too_long ? -1 : (int)o_real;
        __threadfence_system();
        host_out[0] = __float_as_int(prm[6]);
      }
      *done_counter = 0u;
    }
  }
}

// After a mispredicted speculative second phase: the true frame counts back into the arrays the kernels read.
__global__ void restore_lengths_kernel(const int* __restrict__ ylen_real, int* __restrict__ ylen, int* __restrict__ yoff, int B) {
  PDL_LAUNCH();
  PDL_WAIT();
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    int o = 0;
    for (int b = 0; b < B; ++b) {
      ylen[b] = ylen_real[b];
      yoff[b] = o;
      o += ylen_real[b] + (b + 1 < B ? SEQ_GAP : 0);
    }
    yoff[B] = o;
  }
}

// Packed row offsets of the utterances at frame resolution.  SEQ_GAP empty rows separate consecutive utterances
// (never written, zeroed where a TMA-fed kernel reads them) so that a conv halo can never reach a neighbour.
// `host_out` (optional) is pinned host memory mapped into the device address space: the lengths and offsets are
// published there, followed by the call's sequence number (prm[6]), so the host can pick them up by polling instead
// of paying for copy nodes plus a stream synchronisation between the two phases of a call.
__global__ void frame_offsets_kernel(const int* __restrict__ ylen, int* __restrict__ yoff, int B, volatile int* host_out,
                                     const float* __restrict__ prm) {
  PDL_LAUNCH();
  PDL_WAIT();
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    int o = 0;
    for (int b = 0; b < B; ++b) {
      yoff[b] = o;
      if (host_out) { host_out[1 + b] = ylen[b]; host_out[1 + B + b] = o; }
      o += ylen[b] + (b + 1 < B ? SEQ_GAP : 0);
    }
    yoff[B] = o;
    if (host_out) {
      host_out[1 + 2 * B] = o;
      __threadfence_system();
      host_out[0] = __float_as_int(prm[6]);
    }
  }
}

// Split-bf16 planes are read by TMA with a conv halo (and, in the attention, whole key tiles) that reaches past the end of
// an utterance.  Rows outside [0, len) are never written by any producer, but the buffers are reused by calls with other
// lengths, so the rows right behind every utterance of THIS call's layout may hold a previous call's data: they are zeroed
// here, once per phase, for every plane buffer the phase uses (up to ZT_ROWS rows or up to the next utterance's first row;
// the largest halo of the path is 25 rows at >= 4x upsampling where the inter-utterance gap is >= 32 rows, and <= 3 rows at
// frame/token resolution where the gap is SEQ_GAP = 8).  Rows beyond the tensor map's row count read as zero through TMA's
// out-of-bounds fill.  This replaces per-call memsets of whole planes and lets captured graphs serve any length in a bucket.
constexpr int ZT_ROWS = 32, ZT_MAXP = 56;
struct TailList {
  struct E { __nv_bfloat16* hi; __nv_bfloat16* lo; __nv_bfloat16* mid; int C, rm, extra, rows_cap; } e[ZT_MAXP];
  int n;
};
__global__ void zero_tails_kernel(const __grid_constant__ TailList tl, const int* __restrict__ lens, const int* __restrict__ offs, int B) {
  PDL_LAUNCH();
  PDL_WAIT();
  const TailList::E& e = tl.e[blockIdx.x];
  const int b = blockIdx.y;
  // rows behind utterance b: [end, end + ZT_ROWS) -- and, when another utterance follows, also the ZT_ROWS rows in front of
  // ITS first row (its convs' leading halo); a gap of up to 2 * ZT_ROWS rows is simply cleared as a whole
  const long end = ((long)offs[b] + lens[b]) * e.rm + (long)(b + 1) * e.extra;
  long a0 = end, a1 = end + ZT_ROWS, b0 = 0, b1 = 0;
  if (b + 1 < B) {
    const long next = (long)offs[b + 1] * e.rm + (long)(b + 1) * e.extra;
    if (next - end <= 2 * ZT_ROWS) a1 = next;
    else { b0 = next - ZT_ROWS; b1 = next; }
  }
  a1 = min(a1, (long)e.rows_cap);
  b1 = min(b1, (long)e.rows_cap);
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
  for (int part = 0; part < 2; ++part) {
    const long r0 = part ? b0 : a0, r1 = part ? b1 : a1;
    const long n8 = (r1 - r0) * e.C / 8;           // C % 8 == 0: rows are 16-byte multiples
    if (n8 <= 0) continue;
    uint4* ph = reinterpret_cast<uint4*>(e.hi + r0 * e.C);
    uint4* pl = reinterpret_cast<uint4*>(e.lo + r0 * e.C);
    for (long i = threadIdx.x; i < n8; i += blockDim.x) { ph[i] = z; pl[i] = z; }
    if (e.mid) {
      uint4* pm = reinterpret_cast<uint4*>(e.mid + r0 * e.C);
      for (long i = threadIdx.x; i < n8; i += blockDim.x) pm[i] = z;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Length regulator + prior sampling (models.py:1692-1700; commons.generate_path commons.py:128-143):
// frame j takes token idx = #{i : cum_i <= j};  z_p = m_p[idx] + eps * exp(logs_p[idx]) * noise_scale.
// stats rows hold [m_p | logs_p] (enc_p.proj output, models.py:323-325).
// ------------------------------------------------------------------------------------------------
__global__ void sample_prior_kernel(const float* __restrict__ stats, int I, const int* __restrict__ cum,
                                    const int* __restrict__ tok_len, const int* __restrict__ tok_off,
                                    const int* __restrict__ frm_len, const int* __restrict__ frm_off,
                                    const float* __restrict__ eps, int eps_ld, const float* __restrict__ prm,
                                    float* __restrict__ zp, int* __restrict__ frame_token) {
  PDL_LAUNCH();
  PDL_WAIT();
  const uint64_t seed = prm_seed(prm);
  const float noise_scale = prm[0];
  const int b = blockIdx.y;
  const int j = blockIdx.x;
  if (j >= frm_len[b]) return;
  const int T = tok_len[b];
  const int* cb = cum + tok_off[b];
  int lo = 0, hi = T;  // first i with cum[i] > j
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (cb[mid] > j) hi = mid; else lo = mid + 1;
  }
  const int idx = lo;
  const long frow = (long)frm_off[b] + j;
  if (threadIdx.x == 0 && frame_token) frame_token[frow] = idx;
  const bool ok = idx < T;
  const float* srow = stats + ((long)tok_off[b] + (ok ? idx : 0)) * (2 * I);
  for (int c = threadIdx.x; c < I; c += blockDim.x) {
    const float m = ok ? srow[c] : 0.f;
    const float ls = ok ? srow[I + c] : 0.f;
    const float e = eps ? eps[((long)b * I + c) * eps_ld + j] : philox_normal(seed, 2u, (uint32_t)j, (uint32_t)(b * I + c));
    zp[frow * I + c] = __fadd_rn(m, __fmul_rn(__fmul_rn(e, expf(ls)), noise_scale));
  }
}

// MRF mean (models.py:1030-1036): out = (a + b + c ...) / n over up to 3 resblock outputs.
__global__ void mrf_mean_kernel(const float* __restrict__ a, const float* __restrict__ b2, const float* __restrict__ c, int n,
                                float* __restrict__ out, long total4) {
  PDL_LAUNCH();
  PDL_WAIT();
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  float4 s = reinterpret_cast<const float4*>(a)[i];
  if (n > 1) {
    const float4 u = reinterpret_cast<const float4*>(b2)[i];
    s.x += u.x; s.y += u.y; s.z += u.z; s.w += u.w;
  }
  if (n > 2) {
    const float4 u = reinterpret_cast<const float4*>(c)[i];
    s.x += u.x; s.y += u.y; s.z += u.z; s.w += u.w;
  }
  const float d = (float)n;
  s.x /= d; s.y /= d; s.z /= d; s.w /= d;
  reinterpret_cast<float4*>(out)[i] = s;
}

// ------------------------------------------------------------------------------------------------
// MB-iSTFT tail (models.py:1041-1054): spec = exp(.), phase = pi*sin(.), inverse STFT as a transposed
// conv with the fixed basis (stft.py:246-262, no window-sum normalisation), PQMF synthesis
// (pqmf.py:105-116: zero-stuffing x subbands, 63-tap FIR).  One CTA produces TL_M subband samples
// (= TL_M*subbands output samples) of one utterance.
//   post rows: per utterance L1 = 16*Ty + 1 frames of `subbands*(n_fft+2)` channels.
//   w2: null for OnnxSTFT.inverse (VITS2); else the squared window [nfft], and every sample is divided by the window
//       envelope sum_f w2[pos] over the frames that cover it -- torch.istft, as QuickVC's TorchSTFT.inverse calls it
//       (vc/stft.py:197-202).
// ------------------------------------------------------------------------------------------------
constexpr int TL_M = 64;        // subband samples per CTA (256 output samples): 4x more CTAs than the first version, 40 -> ~12 us at batch 1
constexpr int TL_THREADS = 256;
// frames of conv_post output one CTA stages: its TL_M subband samples plus the filter halo on both sides ((taps-1)/2 output
// samples = (taps-1)/2/subbands + 1 subband samples) plus the n_fft-sample reach of a frame, at `hop` samples per frame
__host__ __device__ constexpr int tl_halo(int taps, int subbands) { return (taps - 1) / 2 / subbands + 1; }
__host__ __device__ constexpr int tl_rec_frames(int taps, int subbands, int nfft, int hop) {
  return (TL_M + 2 * tl_halo(taps, subbands) + nfft) / hop + 2;
}

__global__ void __launch_bounds__(TL_THREADS)
istft_pqmf_kernel(const float* __restrict__ post, int ldp, const float* __restrict__ basis, const float* __restrict__ pqmf,
                  int subbands, int nfft, int hop, int taps, int up_total /* frames -> post rows multiplier */,
                  const int* __restrict__ frm_len, const int* __restrict__ frm_off, float* __restrict__ wav, long wav_ld,
                  int packed_out, const float* __restrict__ w2) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y;
  const int Ty = frm_len[b];
  const int L1 = Ty * up_total + 1;            // post-conv frames
  const int M = (L1 - 1) * hop;                // subband samples after trimming nfft/2 on both sides
  const int m0 = blockIdx.x * TL_M;
  if (m0 >= M) return;
  const int nbins = nfft / 2 + 1;
  const int cps = 2 * nbins;                   // channels per subband (18)
  const int halo = (taps - 1) / 2 / subbands + 1;   // subband samples needed on each side (8)
  const int ms = m0 - halo, me = min(M, m0 + TL_M) + halo;     // y range [ms, me)
  // frames contributing to y[m]: 4f <= m + nfft/2 < 4f + nfft
  int f_lo = (ms + nfft / 2 - (nfft - 1));
  f_lo = f_lo <= 0 ? 0 : (f_lo + hop - 1) / hop;
  int f_hi = (me - 1 + nfft / 2) / hop;
  if (f_hi > L1 - 1) f_hi = L1 - 1;
  const int nf = f_hi - f_lo + 1;
  extern __shared__ float sm[];
  float* rec = sm;                                   // [nf][subbands*cps]  (re[0..nbins) | im[0..nbins)) per subband
  float* ysub = rec + (size_t)tl_rec_frames(taps, subbands, nfft, hop) * subbands * cps;   // [subbands][TL_M + 2*halo]
  const int yw = TL_M + 2 * halo;
  const long prow0 = (long)frm_off[b] * up_total + b;
  for (int i = threadIdx.x; i < nf * subbands * nbins; i += TL_THREADS) {
    const int f = i / (subbands * nbins);
    const int r = i - f * subbands * nbins;
    const int k = r / nbins, c = r - k * nbins;
    const float* pr = post + (prow0 + f_lo + f) * (long)ldp + k * cps;
    const float mag = expf(pr[c]);
    const float ph = 3.14159265358979323846f * sinf(pr[nbins + c]);
    float sn, cs;
    sincosf(ph, &sn, &cs);
    rec[(f * subbands + k) * cps + c] = mag * cs;
    rec[(f * subbands + k) * cps + nbins + c] = mag * sn;
  }
  __syncthreads();
  const float scale = (float)nfft / (float)hop;
  for (int i = threadIdx.x; i < subbands * (me - ms); i += TL_THREADS) {
    const int k = i / (me - ms);
    const int m = ms + (i - k * (me - ms));
    float a = 0.f;
    if (m >= 0 && m < M) {
      const int u = m + nfft / 2;
      int fa = u - (nfft - 1);
      fa = fa <= 0 ? 0 : (fa + hop - 1) / hop;
      int fb = u / hop;
      if (fb > L1 - 1) fb = L1 - 1;
      float env = 0.f;
      for (int f = fa; f <= fb; ++f) {
        const float* rr = rec + ((f - f_lo) * subbands + k) * cps;
        const int pos = u - f * hop;
        for (int c = 0; c < cps; ++c) a = fmaf(rr[c], basis[c * nfft + pos], a);
        if (w2) env += w2[pos];
      }
      if (w2) a *= scale / env;          // (env >= 1.25 on every kept sample: no division by a vanishing envelope)
      else a *= scale;
    }
    ysub[k * yw + (m - ms)] = a;
  }
  __syncthreads();
  const int ntap = taps;  // 63
  const int pad = (taps - 1) / 2;
  const int n0 = m0 * subbands, n1 = min(M, m0 + TL_M) * subbands;
  float* wout = packed_out ? (wav + (long)frm_off[b] * up_total * hop * subbands) : (wav + (long)b * wav_ld);
  for (int n = n0 + threadIdx.x; n < n1; n += TL_THREADS) {
    float a = 0.f;
    // up[v] = subbands * y[v/subbands] when v % subbands == 0; out[n] = sum_k sum_j h[k][j] * up_k[n + j - pad]
    const int vlo = n - pad;
    int j0 = ((-vlo) % subbands + subbands) % subbands;   // first j with (vlo + j) % subbands == 0
    for (int j = j0; j < ntap; j += subbands) {
      const int v = vlo + j;
      if (v < 0) continue;
      const int m = v / subbands;
      if (m >= M) break;
      for (int k = 0; k < subbands; ++k) a = fmaf(pqmf[k * ntap + j], (float)subbands * ysub[k * yw + (m - ms)], a);
    }
    wout[n] = a;
  }
}

// Pulls the weight ranges a call will touch into L2 ahead of their first use (prefetch.global.L2 per 128-byte line).
// The kernel retires as soon as the prefetches are issued; the fills overlap with the kernels that follow, so the
// ~130 MB of weights that the benchmark's L2 flush evicts before every step stop costing a DRAM round trip per layer.
struct PrefRange {
  const char* p;
  unsigned long long bytes;
};
__global__ void l2_prefetch_kernel(const PrefRange* __restrict__ ranges, int n, int first, int last) {
  PDL_LAUNCH();
  for (int r = first + blockIdx.y; r < last && r < n; r += gridDim.y) {
    const char* base = ranges[r].p;
    const unsigned long long lines = (ranges[r].bytes + 127ull) >> 7;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < lines;
         i += (unsigned long long)gridDim.x * blockDim.x)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(base + (i << 7)));
  }
}

// int64 -> int32 packing of ids, on device (for the *_dev entry points)
__global__ void pack_ids_kernel(const int64_t* __restrict__ ids, int t_max, int* __restrict__ out, const int* __restrict__ lens,
                                const int* __restrict__ offs) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= lens[b]) return;
  out[offs[b] + t] = (int)ids[(long)b * t_max + t];
}
__global__ void cast_sid_kernel(const int64_t* __restrict__ sid, int* __restrict__ out, int B) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) out[i] = (int)sid[i];
}

}  // namespace vtts
