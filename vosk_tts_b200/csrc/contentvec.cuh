// contentvec.cuh -- the kernels of ContentVec (HubertModel, hubert-base shape, as vc/contentvec.py builds it) that the dense
// conv and attention kernels do not cover: the feature encoder's first layer with its whole-clip GroupNorm, and the
// LayerNorms of width 512 / 768.  Everything here is fp32 FFMA.
//
// Row layout: every clip's rows are contiguous, clip b at offs[b] of its level; the feature encoder's layer-0 rows of clip b
// start at a multiple of 64 (the product of the later strides), so a stride-2 conv over [T][C] rows reads the same memory
// as [T/2][2C] rows and the offsets of every level are exact halvings of the level before.
#pragma once
#include "kernels.cuh"

namespace vtts {

constexpr int CVG_CH = 256;        // layer-0 rows per CTA of the GroupNorm passes
constexpr int CVG_THREADS = 256;
constexpr int CVG_KMAX = 16;       // largest layer-0 kernel

// Layer 0 of the feature encoder, Conv1d(1, C, K0, stride s0, no bias), recomputed from the samples in each pass.  It runs on
// the samples minus the clip's mean mu[b]: without a bias that shifts every channel by a constant, which the GroupNorm removes
// exactly, and a clip with a DC offset then keeps the digits of its signal instead of spending them on the offset.
//   PASS 0: psum[b][j][c] = sum of the chunk's outputs;
//   PASS 1: mean from the clip's chunk sums (fixed order), psq[b][j][c] = sum of (v - mean)^2 over the chunk;
//   PASS 2: out rows = gelu(GroupNorm(v)), GroupNorm with one group per channel over the whole clip (biased variance).
// A clip's statistics are summed in the same order whatever the batch and the grid.  grid (chunks, B).
template <int PASS>
__global__ void __launch_bounds__(CVG_THREADS)
cv_gn_kernel(const float* __restrict__ wav, const float* __restrict__ mu, const int* __restrict__ woff, const int* __restrict__ len0, const int* __restrict__ off0,
             const float* __restrict__ w0, int C, int K0, int s0, float* __restrict__ psum, float* __restrict__ psq, int MC,
             const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float* __restrict__ out) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y, j = blockIdx.x;
  const int L = len0[b];
  const int t0 = j * CVG_CH;
  if (t0 >= L) return;
  const int nt = min(CVG_CH, L - t0);
  const int nch = (L + CVG_CH - 1) / CVG_CH;
  extern __shared__ float xs[];
  const long s_beg = (long)woff[b] + (long)t0 * s0;
  const int ns = (nt - 1) * s0 + K0;
  const float m = mu[b];
  for (int i = threadIdx.x; i < ns; i += CVG_THREADS) xs[i] = wav[s_beg + i] - m;
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += CVG_THREADS) {
    float w[CVG_KMAX];
#pragma unroll
    for (int k = 0; k < CVG_KMAX; ++k) w[k] = k < K0 ? w0[c * K0 + k] : 0.f;
    float mean = 0.f, rstd = 0.f;
    if (PASS >= 1) {
      float s = 0.f;
      for (int q = 0; q < nch; ++q) s += psum[((long)b * MC + q) * C + c];
      mean = s / (float)L;
    }
    if (PASS == 2) {
      float s = 0.f;
      for (int q = 0; q < nch; ++q) s += psq[((long)b * MC + q) * C + c];
      rstd = rsqrtf(s / (float)L + eps);
    }
    const float g = PASS == 2 ? gamma[c] : 0.f, be = PASS == 2 ? beta[c] : 0.f;
    float acc = 0.f;
    for (int t = 0; t < nt; ++t) {
      const float* xp = xs + t * s0;
      float v = 0.f;
#pragma unroll
      for (int k = 0; k < CVG_KMAX; ++k)
        if (k < K0) v = fmaf(w[k], xp[k], v);
      if (PASS == 0) {
        acc += v;
      } else if (PASS == 1) {
        const float d = v - mean;
        acc = fmaf(d, d, acc);
      } else {
        out[((long)off0[b] + t0 + t) * C + c] = gelu_erf(fmaf((v - mean) * rstd, g, be));
      }
    }
    if (PASS == 0) psum[((long)b * MC + j) * C + c] = acc;
    if (PASS == 1) psq[((long)b * MC + j) * C + c] = acc;
  }
}

// LayerNorm of rows up to 1024 wide, one warp per row: out = LN(a + gelu(y)) (y null: LN(a)), two-pass statistics.  Input
// rows at in_offs[b] + t, output rows at out_offs[b] + t (the last layer writes straight into another stage's row layout).
// p_hi / p_lo (or null): the split-bf16 planes of the output rows, the operand of the next tensor-core GEMM.
constexpr int CVL_WARPS = 8;
constexpr int CVL_MAXV = 32;       // values per lane: C <= 1024
__global__ void __launch_bounds__(32 * CVL_WARPS)
cv_ln_kernel(const float* __restrict__ a, const float* __restrict__ y, const float* __restrict__ g, const float* __restrict__ bt, float eps,
             float* __restrict__ out, const int* __restrict__ lens, const int* __restrict__ in_offs, const int* __restrict__ out_offs, int C,
             __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * CVL_WARPS + warp;
  if (t >= lens[b]) return;
  const long ri = ((long)in_offs[b] + t) * C, ro = ((long)out_offs[b] + t) * C;
  float v[CVL_MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < CVL_MAXV; ++i) {
    const int c = lane + 32 * i;
    float u = 0.f;
    if (c < C) {
      u = a[ri + c];
      if (y) u += gelu_erf(y[ri + c]);
    }
    v[i] = u;
    s += u;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < CVL_MAXV; ++i) {
    const int c = lane + 32 * i;
    if (c < C) {
      const float d = v[i] - mean;
      q = fmaf(d, d, q);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)C + eps);
#pragma unroll
  for (int i = 0; i < CVL_MAXV; ++i) {
    const int c = lane + 32 * i;
    if (c < C) {
      const float o = fmaf((v[i] - mean) * rstd, g[c], bt[c]);
      out[ro + c] = o;
      if (p_hi) split_bf16(o, p_hi[ro + c], p_lo[ro + c]);
    }
  }
}

// GELU of the rows of every clip (C channels per row), after a conv: in place, or (p_hi non-null) into split-bf16 planes, the
// operand of the next tensor-core GEMM.  A separate pass rather than an epilogue flag of the conv kernels: an activation
// added to their epilogues slows every other launch of them.  grid (rows, B).
__global__ void __launch_bounds__(256)
cv_gelu_kernel(float* __restrict__ y, int C, const int* __restrict__ lens, const int* __restrict__ offs,
               __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= lens[b]) return;
  const long r = ((long)offs[b] + t) * C;
  for (int c = threadIdx.x; c < C; c += 256) {
    const float g = gelu_erf(y[r + c]);
    if (p_hi) split_bf16(g, p_hi[r + c], p_lo[r + c]);
    else y[r + c] = g;
  }
}

}  // namespace vtts
