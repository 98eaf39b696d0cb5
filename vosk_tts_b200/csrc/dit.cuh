// dit.cuh -- the kernels of the StableTTS flow-matching decoder (CFM.forward -> solve_euler -> Decoder of
// training/stabletts/matcha/models/components/{flow_matching,decoder,diffusion_transformer}.py) that the dense conv and
// attention kernels do not cover: the conditioning rows (time embedding -> FiLM, adaLN-Zero), FiLM + LayerNorm + modulate,
// the rotary embedding, SiLU, the gated residual and the Euler / guidance update.  Everything here is fp32.
//
// Row layout: sequence s of a call occupies rows offs[s] .. offs[s] + lens[s]; with guidance the unconditional branch of
// utterance b is sequence B + b of the same ragged batch, so every launch serves both branches.
#pragma once
#include "kernels.cuh"

namespace vtts {

constexpr int DIT_MAXC = 1024;     // widest hidden / filter width of the conditioning kernels' shared rows
constexpr int DIT_LN_WARPS = 8;
constexpr int DIT_LN_MAXV = 16;    // values per lane of the LayerNorm kernel: hidden <= 512

__device__ __forceinline__ float silu(float v) { return v / (1.f + expf(-v)); }

// out[r] = W[r] . x + b[r] for r in [0, R), W row-major [R][K] (nn.Linear's layout), x in shared memory.  One warp per
// row, lane l sums k = l, l + 32, ... in order and the lanes are reduced by a fixed butterfly: a row's value does not depend
// on the grid or on which other rows are computed beside it.
__device__ __forceinline__ void dit_gemv(const float* __restrict__ W, const float* __restrict__ b, const float* xs, int R, int K,
                                         float* out, bool act) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int r = warp; r < R; r += nw) {
    const float* w = W + (long)r * K;
    float a = 0.f;
    for (int k = lane; k < K; k += 32) a = fmaf(w[k], xs[k], a);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) {
      a += b[r];
      out[r] = act ? silu(a) : a;
    }
  }
}

// FiLM rows of every Euler step in one launch (decoder.py:19-33,35-62,120): CTA k embeds t_k (SinusoidalPosEmb, scale 1000),
// runs time_mlp (Linear, SiLU, Linear) and the 1x1 film conv of each of the NL blocks.  ts[k]: the step's time (fp32, as the
// reference accumulates it); film: [steps][NL][2H] = (gamma | beta).  tw1 [F][H], tw2 [H][F], fw [NL][2H][H].
__global__ void __launch_bounds__(256)
dit_time_kernel(const float* __restrict__ ts, const float* __restrict__ tw1, const float* __restrict__ tb1, const float* __restrict__ tw2,
                const float* __restrict__ tb2, const float* __restrict__ fw, const float* __restrict__ fb, int H, int F, int NL,
                float* __restrict__ film) {
  PDL_LAUNCH();
  PDL_WAIT();
  __shared__ float emb[DIT_MAXC], hid[DIT_MAXC], te[DIT_MAXC];
  const int k = blockIdx.x, half = H / 2;
  const float t = ts[k];
  // the angle in the reference's fp32 steps (1000 t, times the fp32 frequency); exp, sin and cos of those fp32 values are
  // evaluated in double and rounded once: angles reach 1000 rad, where an ulp of the frequency is 1e-4 rad
  const float step = (float)(log(10000.0) / (double)(half - 1));
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    const float a = __fmul_rn(__fmul_rn(1000.f, t), (float)exp((double)__fmul_rn((float)i, -step)));
    emb[i] = (float)sin((double)a);
    emb[half + i] = (float)cos((double)a);
  }
  __syncthreads();
  dit_gemv(tw1, tb1, emb, F, H, hid, true);
  __syncthreads();
  dit_gemv(tw2, tb2, hid, H, F, te, false);
  __syncthreads();
  dit_gemv(fw, fb, te, NL * 2 * H, H, film + (long)k * NL * 2 * H, false);
}

// adaLN-Zero rows (diffusion_transformer.py:107-111,124): grid (NL, sequences).  c = spk_rows[s] (caller embeddings, when
// given and sid[s] >= 0), emb[sid[s]], or the fake speaker (sid[s] < 0: the unconditional branch); out[s][l] =
// W2 . SiLU(W1 . c + b1) + b2, the six chunks shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp of H each.
__global__ void __launch_bounds__(256)
dit_ada_kernel(const float* __restrict__ emb, const float* __restrict__ fake, const float* __restrict__ spk_rows, const int* __restrict__ sid,
               const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
               int G, int H, int NL, int n_spk, float* __restrict__ out) {
  PDL_LAUNCH();
  PDL_WAIT();
  __shared__ float c[DIT_MAXC], hid[DIT_MAXC];
  const int l = blockIdx.x, s = blockIdx.y;
  const int id = sid[s];
  const float* src = id < 0 ? fake : (spk_rows ? spk_rows + (long)s * G : emb + (long)min(id, n_spk - 1) * G);
  for (int i = threadIdx.x; i < G; i += blockDim.x) c[i] = src[i];
  __syncthreads();
  dit_gemv(w1 + (long)l * H * G, b1 + (long)l * H, c, H, G, hid, true);
  __syncthreads();
  dit_gemv(w2 + (long)l * 6 * H * H, b2 + (long)l * 6 * H, hid, 6 * H, H, out + ((long)s * NL + l) * 6 * H, false);
}

// Start of a call (flow_matching.py:52, 186-187) over every sequence's extent exts[s] >= lens[s] (the columns the reference
// pads the frame axis to, matcha_tts.py:162-165; == lens[s] for a decoder called on its own): x = noise * temperature into
// columns [0, NC) of the in_proj operand rows xc [rows][ldx] of both branches, noise from the caller ([rows of the B
// utterances][NC]) or Philox(seed) keyed by (utterance, frame, channel); and fake_content repeated over the frames of the
// unconditional sequences' mu rows.  Rows [lens[s], exts[s]): the conditional mu rows are zeroed, and so is the x half of
// the last long-skip operand skx [rows][2 HC], whose skip half in_proj fills there.  prm[0] temperature, prm[4..5] seed.
// grid (frames, sequences).
__global__ void __launch_bounds__(128)
dit_init_kernel(const float* __restrict__ noise, const float* __restrict__ prm, const float* __restrict__ fake_content, float* __restrict__ xc,
                int ldx, int NC, float* __restrict__ mu, int MC, float* __restrict__ skx, int HC, const int* __restrict__ lens,
                const int* __restrict__ exts, const int* __restrict__ offs, int B) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int s = blockIdx.y, t = blockIdx.x;
  if (t >= exts[s]) return;
  const int b = s < B ? s : s - B;
  const long row = (long)offs[s] + t, nrow = (long)offs[b] + t;
  const float temp = prm[0];
  const uint64_t seed = prm_seed(prm);
  for (int c = threadIdx.x; c < NC; c += blockDim.x) {
    const float e = noise ? noise[nrow * NC + c] : philox_normal(seed, 7u, (uint32_t)t, (uint32_t)(b * NC + c));
    xc[row * ldx + c] = e * temp;
  }
  if (s >= B)
    for (int c = threadIdx.x; c < MC; c += blockDim.x) mu[row * MC + c] = fake_content[c];
  if (t >= lens[s]) {
    if (s < B)
      for (int c = threadIdx.x; c < MC; c += blockDim.x) mu[row * MC + c] = 0.f;
    for (int c = threadIdx.x; c < HC; c += blockDim.x) skx[row * 2 * HC + c] = 0.f;
  }
}

// cos / sin of the rotary embedding (diffusion_transformer.py:151-166) for positions [0, n): theta_i = 1 / 10000^(2i/d) in
// fp32, the fp32 product with the position, then cos / sin of that fp32 angle, evaluated in double and rounded once, so
// that large positions carry no range-reduction error of their own.  tab [n][d/2] (cos, sin).
__global__ void __launch_bounds__(128)
dit_rope_table_kernel(float2* __restrict__ tab, int n, int d) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int hd = d / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * hd) return;
  const int pos = i / hd, j = i - pos * hd;
  const float theta = 1.f / powf(10000.f, (float)(2 * j) / (float)d);
  const float a = __fmul_rn((float)pos, theta);
  tab[i] = make_float2((float)cos((double)a), (float)sin((double)a));
}

// Rotary embedding of q and k in place on the qkv rows [rows][3 * heads * dk] (diffusion_transformer.py:81-82,179-197): the
// first d features of each head are rotated, pair (j, j + d/2): x_j cos - x_{j+d/2} sin, x_{j+d/2} cos + x_j sin, as two
// rounded products and a rounded sum like the reference; the other dk - d pass through.  grid (frames, sequences).
__global__ void __launch_bounds__(128)
dit_rope_kernel(float* __restrict__ qkv, const float2* __restrict__ tab, int heads, int dk, int d, const int* __restrict__ lens,
                const int* __restrict__ offs) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int s = blockIdx.y, t = blockIdx.x;
  if (t >= lens[s]) return;
  const int hd = d / 2, HT = heads * dk;
  float* row = qkv + ((long)offs[s] + t) * 3 * HT;
  for (int i = threadIdx.x; i < 2 * heads * hd; i += blockDim.x) {
    const int j = i % hd, hq = i / hd;          // hq: head of q, then head of k
    float* p = row + (hq / heads) * HT + (hq % heads) * dk;
    const float2 cs = tab[(long)t * hd + j];
    const float a = p[j], b = p[j + hd];
    p[j] = __fadd_rn(__fmul_rn(a, cs.x), __fmul_rn(-b, cs.y));
    p[j + hd] = __fadd_rn(__fmul_rn(b, cs.x), __fmul_rn(a, cs.y));
  }
}

// v = a (FiLM: gamma * a + beta, decoder.py:16,33) (+ gate * y: the gated attention residual, diffusion_transformer.py:112);
// xo = v; no = LayerNorm(v) * (1 + scale) + shift without affine (:100,102,120-121), two-pass statistics, one warp per row.
// film: (gamma | beta) [2C] of the step and block, or null.  gate / shift / scale: rows of the sequence's adaLN block
// ada + s * ada_ld.  a rows have pitch lda (the residual stream lives in column blocks of the long-skip operands).
__global__ void __launch_bounds__(32 * DIT_LN_WARPS)
dit_norm_kernel(const float* __restrict__ a, int lda, const float* __restrict__ film, const float* __restrict__ y, const float* __restrict__ ada,
                int ada_ld, int gate_off, int shift_off, int scale_off, float eps, float* __restrict__ xo, float* __restrict__ no,
                const int* __restrict__ lens, const int* __restrict__ offs, int C) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int s = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * DIT_LN_WARPS + warp;
  if (t >= lens[s]) return;
  const long r = (long)offs[s] + t;
  const float* ad = ada + (long)s * ada_ld;
  float v[DIT_LN_MAXV];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < DIT_LN_MAXV; ++i) {
    const int c = lane + 32 * i;
    float u = 0.f;
    if (c < C) {
      u = a[r * lda + c];
      if (film) u = __fadd_rn(__fmul_rn(film[c], u), film[C + c]);
      if (y) u = __fadd_rn(u, __fmul_rn(ad[gate_off + c], y[r * C + c]));
      xo[r * C + c] = u;
    }
    v[i] = u;
    sum += u;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < DIT_LN_MAXV; ++i) {
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
  for (int i = 0; i < DIT_LN_MAXV; ++i) {
    const int c = lane + 32 * i;
    if (c < C) no[r * C + c] = __fadd_rn(__fmul_rn((v[i] - mean) * rstd, 1.f + ad[scale_off + c]), ad[shift_off + c]);
  }
}

// SiLU of the rows of every sequence in place, after a conv (a separate pass rather than an epilogue flag of the conv
// kernels, like cv_gelu_kernel).  grid (frames, sequences).
__global__ void __launch_bounds__(256)
dit_silu_kernel(float* __restrict__ y, int C, const int* __restrict__ lens, const int* __restrict__ offs) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int s = blockIdx.y, t = blockIdx.x;
  if (t >= lens[s]) return;
  float* r = y + ((long)offs[s] + t) * C;
  for (int c = threadIdx.x; c < C; c += 256) r[c] = silu(r[c]);
}

// Gated residual of the FFN (diffusion_transformer.py:113): out = x + gate * y, out rows of pitch ldo (a column block of a
// long-skip operand, or plain rows).  grid (frames, sequences).
__global__ void __launch_bounds__(128)
dit_gate_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ ada, int ada_ld, int gate_off,
                float* __restrict__ out, int ldo, const int* __restrict__ lens, const int* __restrict__ offs, int C) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int s = blockIdx.y, t = blockIdx.x;
  if (t >= lens[s]) return;
  const long r = (long)offs[s] + t;
  const float* g = ada + (long)s * ada_ld + gate_off;
  for (int c = threadIdx.x; c < C; c += 128) out[r * ldo + c] = __fadd_rn(x[r * C + c], __fmul_rn(g[c], y[r * C + c]));
}

// One Euler step with classifier-free guidance (flow_matching.py:93-94,182-194): d = v_c + s (v_c - v_u) (s = 0: d = v_c,
// no unconditional sequence), x <- x + dt d, written to the x columns of both branches' in_proj operand rows.  The last step
// (mel non-null) also writes the result rows [rows of the B utterances][NC], times mel_std plus mel_mean when prm[2] != 0.
// prm[1] = s; dt: this step's.  grid (frames, B).
__global__ void __launch_bounds__(128)
dit_euler_kernel(const float* __restrict__ v, float* __restrict__ xc, int ldx, int NC, const float* __restrict__ dt, const float* __restrict__ prm,
                 int guided, float* __restrict__ mel, const float* __restrict__ mel_mean, const float* __restrict__ mel_std,
                 const int* __restrict__ lens, const int* __restrict__ offs, int B) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= lens[b]) return;
  const long rc = (long)offs[b] + t, ru = guided ? (long)offs[B + b] + t : 0;
  const float h = dt[0], s = prm[1];
  const bool den = prm[2] != 0.f;
  for (int c = threadIdx.x; c < NC; c += blockDim.x) {
    float d = v[rc * NC + c];
    if (guided) d = __fadd_rn(d, __fmul_rn(s, __fadd_rn(d, -v[ru * NC + c])));
    const float x = __fadd_rn(xc[rc * ldx + c], __fmul_rn(h, d));
    xc[rc * ldx + c] = x;
    if (guided) xc[ru * ldx + c] = x;
    if (mel) mel[rc * NC + c] = den ? __fadd_rn(__fmul_rn(x, mel_std[0]), mel_mean[0]) : x;
  }
}

// Precision mode 2 (the mel phase's convs and attention on the tensor cores): the kernels above that feed a wgmma operand,
// writing the same fp32 rows and also the split-bf16 planes of their output.  Defined in st_tc.cu, a translation unit of
// its own: see there.
__global__ void dit_norm_planes_kernel(const float* __restrict__ a, int lda, const float* __restrict__ film, const float* __restrict__ y,
                                       const float* __restrict__ ada, int ada_ld, int gate_off, int shift_off, int scale_off, float eps,
                                       float* __restrict__ xo, float* __restrict__ no, __nv_bfloat16* __restrict__ p_hi,
                                       __nv_bfloat16* __restrict__ p_lo, const int* __restrict__ lens, const int* __restrict__ offs, int C);
__global__ void dit_rope_planes_kernel(float* __restrict__ qkv, const float2* __restrict__ tab, int heads, int dk, int d,
                                       __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo, const int* __restrict__ lens,
                                       const int* __restrict__ offs);
__global__ void dit_silu_planes_kernel(float* __restrict__ y, int C, __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo,
                                       const int* __restrict__ lens, const int* __restrict__ offs);
__global__ void dit_gate_planes_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ ada, int ada_ld,
                                       int gate_off, float* __restrict__ out, int ldo, __nv_bfloat16* __restrict__ p_hi,
                                       __nv_bfloat16* __restrict__ p_lo, const int* __restrict__ lens, const int* __restrict__ offs, int C);

}  // namespace vtts
