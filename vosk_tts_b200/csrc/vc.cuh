// vc.cuh -- kernels of the voice-conversion path (SynthesizerTrn.voice_conversion, training/vits2/models.py:1710-1718) that
// the TTS path does not have: the spectrogram front end (mel_processing.py:53-125), the posterior sampling of enc_q
// (models.py:836-842) and the two-speaker conditioning launch.  The posterior encoder's WN, both flow directions and the
// decoder run on the conv kernels of kernels.cuh / conv_tc.cuh.
//
// Layout as everywhere else: channels-last packed rows, clip b occupies frame rows [off[b], off[b] + len[b]).
#pragma once
#include "kernels.cuh"

namespace vtts {

// ------------------------------------------------------------------------------------------------
// Conditioning of both speakers in ONE launch: rows [0, R) of the stacked TTS matrix (spk_emb_linear, dp.cond, the flow's
// WN cond_layers, dec.cond) for g_src and g_tgt, plus the Rq rows of enc_q's WN cond_layer for g_src only.
//   sid: [2B] (sources, then targets);  out_src: [B][R + Rq];  out_tgt: [B][R]
// Same arithmetic as cond_kernel, so a speaker's rows come out bit-identical whichever side they were computed for.
// ------------------------------------------------------------------------------------------------
__global__ void cond_vc_kernel(const float* __restrict__ emb_g, const int* __restrict__ sid, const float* __restrict__ W,
                               const float* __restrict__ bias, int R, const float* __restrict__ Wq, const float* __restrict__ bq,
                               int Rq, float* __restrict__ out_src, float* __restrict__ out_tgt, int G, int B, int n_speakers) {
  PDL_LAUNCH();
  PDL_WAIT();
  extern __shared__ float gs[];
  const int y = blockIdx.y;
  const bool src = y < B;
  const int b = src ? y : y - B;
  int s = sid[y];
  s = s < 0 ? 0 : (s >= n_speakers ? n_speakers - 1 : s);      // (the host rejects out-of-range ids)
  for (int i = threadIdx.x; i < G; i += blockDim.x) gs[i] = emb_g[(long)s * G + i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + warp;
  if (r >= (src ? R + Rq : R)) return;
  const float* wr = r < R ? W + (long)r * G : Wq + (long)(r - R) * G;
  float a = 0.f;
  for (int i = lane; i < G; i += 32) a = fmaf(wr[i], gs[i], a);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (lane == 0) {
    const float v = a + (r < R ? bias[r] : bq[r - R]);
    if (src) out_src[(long)b * (R + Rq) + r] = v;
    else out_tgt[(long)b * R + r] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// Magnitude spectrogram (spectrogram_torch, mel_processing.py:53-77): reflect padding by `padl` on both sides, frames of
// n_fft samples every `hop` (center=False), periodic Hann window, sqrt(re^2 + im^2 + 1e-6).
// The DFT is a fp32 GEMM  S[t][c] = sum_n xpad[t*hop + n] * basis[n][c]  against a windowed basis whose column pairs
// (2k, 2k+1) hold (cos, sin) of bin k; sin of bin 0 is identically zero, so column 1 carries the cosine of the Nyquist bin
// instead (weights.stft_basis).  The reflect padding is folded into the operand load: every clip is padded on its own samples.
// One CTA = 64 frames x 64 basis columns (32 bins) of one clip; 256 threads, 4 x 4 outputs each.
// Output: out[row][k] for k < n_fft/2 + 1, zeros in the pad columns up to ldo.
// ------------------------------------------------------------------------------------------------
constexpr int ST_TM = 64, ST_TN = 64, ST_TK = 16, ST_THREADS = 256;

__global__ void __launch_bounds__(ST_THREADS)
stft_mag_kernel(const float* __restrict__ wav, long wav_ld, const int* __restrict__ clip_len, const float* __restrict__ basis,
                int nfft, int hop, int padl, const int* __restrict__ frm_len, const int* __restrict__ frm_off, float* __restrict__ out,
                int ldo) {
  PDL_LAUNCH();
  PDL_WAIT();
  __shared__ float As[ST_TK][ST_TM + 4];
  __shared__ __align__(16) float Bs[ST_TK][ST_TN];
  const int b = blockIdx.z;
  const int F = frm_len[b];
  const int t0 = blockIdx.x * ST_TM;
  if (t0 >= F) return;
  const int c0 = blockIdx.y * ST_TN;
  const int L = clip_len[b];
  const float* x = wav + (long)b * wav_ld;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < nfft; k0 += ST_TK) {
    for (int i = tid; i < ST_TK * ST_TM; i += ST_THREADS) {
      const int kk = i / ST_TM, tt = i % ST_TM, t = t0 + tt;
      float v = 0.f;
      if (t < F) {
        int q = t * hop + k0 + kk - padl;
        if (q < 0) q = -q;                       // ReflectionPad (mel_processing.py:67)
        if (q >= L) q = 2 * (L - 1) - q;
        v = x[q];
      }
      As[kk][tt] = v;
    }
    for (int i = tid; i < ST_TK * ST_TN / 4; i += ST_THREADS) {
      const int kk = i / (ST_TN / 4), cc = (i % (ST_TN / 4)) * 4;
      *reinterpret_cast<float4*>(&Bs[kk][cc]) = *reinterpret_cast<const float4*>(basis + (long)(k0 + kk) * nfft + c0 + cc);
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < ST_TK; ++kk) {
      float a[4], w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty + 16 * i];
      const float4 w4 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      w[0] = w4.x; w[1] = w4.y; w[2] = w4.z; w[3] = w4.w;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
    }
    __syncthreads();
  }
  const int nbins = nfft / 2 + 1;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int t = t0 + ty + 16 * i;
    if (t >= F) continue;
    float* orow = out + ((long)frm_off[b] + t) * ldo;
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const int k = (c0 + tx * 4) / 2 + p;
      const float re = acc[i][2 * p], im = acc[i][2 * p + 1];
      if (k == 0) {
        orow[0] = sqrtf(__fadd_rn(__fmul_rn(re, re), 1e-6f));
        orow[nbins - 1] = sqrtf(__fadd_rn(__fmul_rn(im, im), 1e-6f));
      } else {
        orow[k] = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im)), 1e-6f));
      }
    }
    if (blockIdx.y == 0 && tx == 0)
      for (int c = nbins; c < ldo; ++c) orow[c] = 0.f;
  }
}

// ------------------------------------------------------------------------------------------------
// Mel projection + log compression (spec_to_mel_torch / spectral_normalize_torch, mel_processing.py:80-90, 36-38):
//   out[row][m] = log(max(sum_k mel[m][k] * spec[row][k], 1e-5)),  pad columns [nmel, ldo) zeroed.
// One CTA = MEL_ROWS frames of one clip; the spectrum rows are staged in shared memory.
// ------------------------------------------------------------------------------------------------
constexpr int MEL_ROWS = 8, MEL_THREADS = 256;
// dynamic shared memory of a launch for n_fft; the engine opts the kernel in to MEL_SMEM_MAX and refuses an n_fft above it
constexpr int MEL_SMEM_MAX = 227 * 1024;
constexpr size_t mel_smem_bytes(int nfft) { return (size_t)MEL_ROWS * (nfft / 2 + 1) * sizeof(float); }

__global__ void __launch_bounds__(MEL_THREADS)
mel_log_kernel(const float* __restrict__ spec, int lds, const float* __restrict__ mel, int nbins, int nmel,
               const int* __restrict__ frm_len, const int* __restrict__ frm_off, float* __restrict__ out, int ldo) {
  PDL_LAUNCH();
  PDL_WAIT();
  extern __shared__ float sp[];          // [MEL_ROWS][nbins]
  const int b = blockIdx.y;
  const int F = frm_len[b];
  const int t0 = blockIdx.x * MEL_ROWS;
  if (t0 >= F) return;
  const long r0 = (long)frm_off[b] + t0;
  const int nr = min(MEL_ROWS, F - t0);
  for (int i = threadIdx.x; i < nr * nbins; i += blockDim.x) {
    const int f = i / nbins, k = i % nbins;
    sp[f * nbins + k] = spec[(r0 + f) * lds + k];
  }
  __syncthreads();
  for (int o = threadIdx.x; o < nr * ldo; o += blockDim.x) {
    const int f = o / ldo, m = o % ldo;
    float v = 0.f;
    if (m < nmel) {
      const float* mr = mel + (long)m * nbins;
      const float* s = sp + f * nbins;
      float a = 0.f;
      for (int k = 0; k < nbins; ++k) a = fmaf(mr[k], s[k], a);
      v = logf(fmaxf(a, 1e-5f));
    }
    out[(r0 + f) * ldo + m] = v;
  }
}

// Caller-supplied features [B][C][ld] (the reference's `y`, models.py:1710) -> packed rows [row][ldo], pad columns zeroed.
__global__ void spec_pack_kernel(const float* __restrict__ in, int C, int ld, const int* __restrict__ frm_len,
                                 const int* __restrict__ frm_off, float* __restrict__ out, int ldo) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= frm_len[b]) return;
  const long row = (long)frm_off[b] + t;
  for (int c = threadIdx.x; c < ldo; c += blockDim.x) out[row * ldo + c] = c < C ? in[((long)b * C + c) * ld + t] : 0.f;
}

// ------------------------------------------------------------------------------------------------
// Posterior sampling (models.py:840-841): z = (m + eps * exp(logs) * noise_scale) * mask, stats rows = [m | logs].
// eps: caller-supplied [B][I][eps_ld], or Philox (stream 3) from the per-call seed.  noise_scale = prm[0]; with 1 the op
// order is the reference's m + eps * exp(logs).  Rows beyond a clip are not written (the mask).
// ------------------------------------------------------------------------------------------------
__global__ void posterior_sample_kernel(const float* __restrict__ stats, int I, const float* __restrict__ eps, int eps_ld,
                                        const float* __restrict__ prm, const int* __restrict__ frm_len,
                                        const int* __restrict__ frm_off, float* __restrict__ z) {
  PDL_LAUNCH();
  PDL_WAIT();
  const uint64_t seed = prm_seed(prm);
  const float noise_scale = prm[0];
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= frm_len[b]) return;
  const long row = (long)frm_off[b] + t;
  const float* srow = stats + row * (2 * I);
  for (int c = threadIdx.x; c < I; c += blockDim.x) {
    const float e = eps ? eps[((long)b * I + c) * eps_ld + t] : philox_normal(seed, 3u, (uint32_t)t, (uint32_t)(b * I + c));
    z[row * I + c] = __fadd_rn(srow[c], __fmul_rn(__fmul_rn(e, expf(srow[I + c])), noise_scale));
  }
}

}  // namespace vtts
