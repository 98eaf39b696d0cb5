// stabletts.cuh -- the kernels of StableTTS text-to-mel around the flow-matching decoder (MatchaTTS.synthesise,
// training/stabletts/matcha/models/matcha_tts.py:93-211; TextEncoder.forward, components/text_encoder.py:109-139): the token
// front (embedding gathers, bert_proj, concatenation), the durations with their scan, the expansion of token rows to frame
// rows and the pause fill.  The two encoder stacks run on the block sequence of the decoder (dit.cuh).  Everything is fp32.
//
// Token rows: utterance b occupies rows tok_off[b] .. tok_off[b] + tok_len[b]; frame rows as in dit.cuh.
#pragma once
#include "dit.cuh"

namespace vtts {

constexpr int STT_MAXBERT = 1024;   // widest BERT feature row the token front stages in shared memory
constexpr int STT_SCAN = 256;       // tokens per pass of the duration scan

// x row of every token (text_encoder.py:111-131): emb[ids[0]] * es (E channels) | punc[ids[s]] * ps for streams 1 .. S-1
// (P channels each, one table) | bert_proj(bert row) (R channels, Linear(BD, R); dit_gemv's fixed summation order).
// ids: [S][token rows]; bert: [token rows][BD]; x: [token rows][E + (S - 1) P + R].  grid (tokens, utterances).
__global__ void __launch_bounds__(256)
stt_front_kernel(const int* __restrict__ ids, int id_ld, const float* __restrict__ bert, const float* __restrict__ emb, float es,
                 const float* __restrict__ punc, float ps, const float* __restrict__ bw, const float* __restrict__ bb, int S, int E, int P, int BD,
                 int R, float* __restrict__ x, const int* __restrict__ lens, const int* __restrict__ offs) {
  PDL_LAUNCH();
  PDL_WAIT();
  __shared__ float br[STT_MAXBERT];
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= lens[b]) return;
  const long r = (long)offs[b] + t;
  const int W = E + (S - 1) * P + R;
  float* row = x + r * W;
  for (int i = threadIdx.x; i < BD; i += blockDim.x) br[i] = bert[r * BD + i];
  const float* e = emb + (long)ids[r] * E;
  for (int c = threadIdx.x; c < E; c += blockDim.x) row[c] = __fmul_rn(e[c], es);
  for (int c = threadIdx.x; c < (S - 1) * P; c += blockDim.x) {
    const int s = 1 + c / P;
    row[E + c] = __fmul_rn(punc[(long)ids[(long)s * id_ld + r] * P + (c - (s - 1) * P)], ps);
  }
  __syncthreads();
  dit_gemv(bw, bb, br, R, BD, row + E + (S - 1) * P, false);
}

// Durations of every token and their scan (matcha_tts.py:143-160), one CTA per utterance: logw = sum over the DC channels of
// sigmoid(mu_dp), summed in channel order by one thread; the pause override where pause != 0; w = max(rint(logw *
// length_scale), 1) (torch.round: half to even), capped at wmax.  Integer from there on: dur[row] = w, first[row] = the
// token's first frame, ylen[b] = the utterance's frames.  prm[0] = length_scale.  logw: the pre-rounding value of each token.
__global__ void __launch_bounds__(STT_SCAN)
stt_dur_kernel(const float* __restrict__ mu_dp, int ld, int DC, const float* __restrict__ pause, const float* __restrict__ prm, float wmax,
               int* __restrict__ dur, int* __restrict__ first, int* __restrict__ ylen, float* __restrict__ logw,
               const int* __restrict__ lens, const int* __restrict__ offs) {
  PDL_LAUNCH();
  PDL_WAIT();
  __shared__ int sc[STT_SCAN];
  const int b = blockIdx.x, n = lens[b], tid = threadIdx.x;
  const long base = offs[b];
  const float ls = prm[0];
  int carry = 0;
  for (int t0 = 0; t0 < n; t0 += STT_SCAN) {
    const int t = t0 + tid;
    int w = 0;
    if (t < n) {
      const float* m = mu_dp + (base + t) * ld;
      float a = 0.f;
      for (int c = 0; c < DC; ++c) a = __fadd_rn(a, 1.f / (1.f + expf(-m[c])));
      const float p = pause[base + t];
      if (p != 0.f) a = p;
      a = __fmul_rn(a, ls);
      logw[base + t] = a;
      w = (int)fminf(fmaxf(rintf(a), 1.f), wmax);
      dur[base + t] = w;
    }
    sc[tid] = w;
    __syncthreads();
    for (int o = 1; o < STT_SCAN; o <<= 1) {
      const int v = tid >= o ? sc[tid - o] : 0;
      __syncthreads();
      sc[tid] += v;
      __syncthreads();
    }
    if (t < n) first[base + t] = carry + sc[tid] - w;
    carry += sc[STT_SCAN - 1];
    __syncthreads();
  }
  if (tid == 0) ylen[b] = carry;
}

// Token rows -> frame rows (generate_path and the three matmuls with it, matcha_tts.py:164-180): token i of utterance b owns
// frames first[i] .. first[i] + dur[i] of the utterance's frame rows.  mu [frame rows][MC] <- x [token rows][MC]; pau [frame
// rows] <- the token's pause; prior [frame rows][PC] <- mu_mel [token rows][PC] (times mel_std plus mel_mean when prm[2] != 0)
// when prior is non-null.  grid (tokens, utterances); (tl, to) token rows, fo frame offsets.
__global__ void __launch_bounds__(128)
stt_expand_kernel(const float* __restrict__ x, int MC, const float* __restrict__ pause, const float* __restrict__ mu_mel, int PC,
                  const int* __restrict__ dur, const int* __restrict__ first, float* __restrict__ mu, float* __restrict__ pau,
                  float* __restrict__ prior, const float* __restrict__ prm, const float* __restrict__ mel_mean, const float* __restrict__ mel_std,
                  const int* __restrict__ tl, const int* __restrict__ to, const int* __restrict__ fo) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= tl[b]) return;
  const long r = (long)to[b] + t, f0 = (long)fo[b] + first[r];
  const int w = dur[r];
  const float p = pause[r];
  const bool den = prm[2] != 0.f;
  for (int f = 0; f < w; ++f) {
    for (int c = threadIdx.x; c < MC; c += blockDim.x) mu[(f0 + f) * MC + c] = x[r * MC + c];
    if (prior)
      for (int c = threadIdx.x; c < PC; c += blockDim.x) {
        const float v = mu_mel[r * PC + c];
        prior[(f0 + f) * PC + c] = den ? __fadd_rn(__fmul_rn(v, mel_std[0]), mel_mean[0]) : v;
      }
    if (threadIdx.x == 0) pau[f0 + f] = p;
  }
}

// Pause frames (matcha_tts.py:186-197): every frame of an utterance whose token carries a pause takes the utterance's own
// frame 0 (the reference, called with one utterance, takes utterance 0's).  In place on the mel rows after the last Euler
// step; denormalisation is elementwise, so filling after it gives the bits of filling before it.  grid (frames, B).
__global__ void __launch_bounds__(128)
stt_pause_fill_kernel(float* __restrict__ mel, int NC, const float* __restrict__ pau, const int* __restrict__ lens, const int* __restrict__ offs) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y, t = blockIdx.x;
  if (t == 0 || t >= lens[b]) return;
  const long r0 = offs[b], r = r0 + t;
  if (!(pau[r] > 0.f)) return;
  for (int c = threadIdx.x; c < NC; c += blockDim.x) mel[r * NC + c] = mel[r0 * NC + c];
}

// Each token's BERT row (vosk_tts/synth.py:25-44 and the word index of g2p_multistream*, :273-454): bert [token rows][BD] <-
// feat [src[token row]][BD], BERT's packed rows of the utterance's own sentence.  grid (tokens, utterances).  Defined in
// st_gather.cu, a translation unit of its own: see there.
__global__ void st_bert_gather_kernel(const float* __restrict__ feat, const int* __restrict__ src, int BD, float* __restrict__ bert,
                                      const int* __restrict__ lens, const int* __restrict__ offs);

}  // namespace vtts
