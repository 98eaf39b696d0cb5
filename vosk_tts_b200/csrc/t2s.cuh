// t2s.cuh -- GPT-SoVITS text-to-semantic decoding (Text2SemanticDecoder.infer_panel, training/gpt-sovits/ar/models/
// t2s_model.py:324-448): the kernels of the text prefill that post_ln_layers does not already hold, and every kernel of the
// one-token decode step and its sampler.  Defined in t2s.cu, a translation unit of its own (as st_gather.cu): engine.cu's
// module keeps exactly the kernels it held before.  fp32 FFMA; DESIGN.md 4.s.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

// Shared memory of a decode GEMV CTA: the input rows [T2S_RB][Cin], then the warp partials [T2S_WARPS][T2S_RB][32].
#define T2S_GEMV_SMEM(Cin) (((size_t)vtts::T2S_RB * (Cin) + vtts::T2S_WARPS * vtts::T2S_RB * 32) * sizeof(float))

namespace vtts {

constexpr int T2S_RB = 4;            // rows (utterances) per CTA of the decode GEMVs
constexpr int T2S_COLS = 32;         // output columns per CTA of the decode GEMVs (one per lane)
constexpr int T2S_WARPS = 32;        // warps per GEMV CTA, each a fixed 32nd of the input width (bytes in flight per SM)
constexpr int T2S_KS = 64;           // keys per CTA of the decode attention: a fixed split, whatever the batch
constexpr int T2S_SAMPLE_THREADS = 1024;
constexpr int T2S_MAX_V = 4096;      // the sampler's block sort holds the vocabulary in shared memory
constexpr int T2S_ST = 8;            // ints of per-utterance state (T2sSt)

// Per-utterance decode state, T2S_ST ints at st[b * T2S_ST]:
enum T2sSt { ST_T = 0, ST_P = 1, ST_KV = 2, ST_NY = 3, ST_GEN = 4, ST_STOP = 5, ST_YOFF = 6 };
//   T text rows, P prompt tokens, KV the utterance's first cache row, NY audio tokens run through the layers so far,
//   GEN tokens sampled so far, STOP 1 once stopped (the row is then frozen), YOFF the first slot of its tokens in y.
// A step runs the layers on token y[NY] (position NY) when NY < P + GEN, then samples token P + GEN once NY == P + GEN.

// Per-call sampling scalars (device memory, so that a captured decode graph serves every call).
struct T2sPrm {
  float top_p, temperature, penalty;
  int top_k, early_stop, step_cap, q_ld, logits_ld;   // q_ld / logits_ld: steps of the caller's q / raw-logit rows (0: none)
};

struct T2sLayer {                   // one post-LN layer's decode weights: W^T rows [in][ldw] (the FFMA conv layout), biases
  const float *wqkv, *bqkv, *wo, *bo, *w1, *b1, *w2, *b2, *ln1g, *ln1b, *ln2g, *ln2b;
  int ldqkv, ldo, ld1, ld2;         // row pitches of the four weights
  float eps;                        // LayerNorm eps
  float* kc;                        // K and V caches of the layer: [cache rows][H]
  float* vc;
};

// ---- prefill of the [text; prompt] rows (the layers themselves are engine.cu post_ln_layers)
// Text row t < T of b: (temb[ids] + bert_proj) + alpha_t * pe[t] (bp null: bert_proj's bias alone, zero BERT features); prompt
// row t >= T: aemb[ids] + alpha_a * pe[t - T].  T = init[b][0].  p_hi: planes.
__global__ void t2s_prefill_embed_kernel(const int* __restrict__ ids, const float* __restrict__ temb, const float* __restrict__ aemb,
                                         const float* __restrict__ bp, const float* __restrict__ bp_bias, const float* __restrict__ pe,
                                         float alpha_t, float alpha_a, int H, float* __restrict__ x, const int* __restrict__ lens,
                                         const int* __restrict__ offs, const int* __restrict__ init, __nv_bfloat16* __restrict__ p_hi,
                                         __nv_bfloat16* __restrict__ p_lo);
// The prefill's attention under infer_panel's prefix mask: row t of b sees key k iff k < T or k <= t (T = init[b][0]; text
// rows see the text only, prompt rows the text and the prompt up to themselves).  qkv rows [rows][3H]; out ao [rows][H] and,
// when p_hi is given, its split-bf16 planes.  grid (rows, heads, B), one warp; dk a multiple of 32 up to 128.
__global__ void t2s_prefix_attn_kernel(const float* __restrict__ qkv, int H, int dk, float scale, float* __restrict__ ao,
                                       const int* __restrict__ lens, const int* __restrict__ offs, const int* __restrict__ init,
                                       __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo);
// ReLU of the FFN rows, in place or into planes (post_ln_layers' activation for this family; cv_gelu_kernel's layout).
__global__ void t2s_relu_kernel(float* __restrict__ y, int C, const int* __restrict__ lens, const int* __restrict__ offs,
                                __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo);
// K and V columns of a layer's packed q | k | v rows into the cache: row (b, t) -> cache row init[b][2] + t.
__global__ void t2s_kv_store_kernel(const float* __restrict__ qkv, int H, float* __restrict__ kc, float* __restrict__ vc,
                                    const int* __restrict__ lens, const int* __restrict__ offs, const int* __restrict__ init);
// State, tokens and seen bitmap of every utterance from init [B][4] (T, P, first cache row, first token slot); hx[b] = the
// last row of the prefill (the first logits' input).  NY starts at P: the prefill ran the layers on the prompt.
__global__ void t2s_init_kernel(const int* __restrict__ init, const int* __restrict__ prompt, const int* __restrict__ poffs,
                                const float* __restrict__ pre, const int* __restrict__ offs, int H, int V, int* __restrict__ st,
                                int* __restrict__ y, unsigned* __restrict__ seen, float* __restrict__ hx);

// ---- one decode step (grids: x column tiles, y row tiles of T2S_RB)
// layer 0: x = audio_emb[y[NY]] + alpha * pe[NY]; layer l > 0: x = LN2_{l-1}(y2 (+ residual already added)).  Writes x (CTA 0),
// q = x Wq + bq, and appends k, v to the cache at row KV + T + NY.
__global__ void t2s_qkv_kernel(T2sLayer L, const float* __restrict__ lnpg, const float* __restrict__ lnpb, const float* __restrict__ aemb,
                               const float* __restrict__ pe, float alpha, const int* __restrict__ y, const float* __restrict__ y2,
                               float* __restrict__ x, float* __restrict__ q, const int* __restrict__ st, int B, int H);
// One head of one utterance over T2S_KS cached keys: partial (max, sum, numerator) at part[((b * heads + h) * nsplit + s)].
__global__ void t2s_attn_kernel(const float* __restrict__ q, const float* __restrict__ kc, const float* __restrict__ vc,
                                float* __restrict__ part, const int* __restrict__ st, int H, int dk, float scale, int nsplit);
// Combines the partials (fixed order), then y1 = attn Wo + bo + x.
__global__ void t2s_o_kernel(T2sLayer L, const float* __restrict__ part, const float* __restrict__ x, float* __restrict__ y1,
                             const int* __restrict__ st, int B, int H, int dk, int nsplit);
// xm = LN1(y1) (CTA 0 writes it), ff = relu(xm W1 + b1).
__global__ void t2s_ffn1_kernel(T2sLayer L, const float* __restrict__ y1, float* __restrict__ xm, float* __restrict__ ff,
                                const int* __restrict__ st, int B, int H, int F);
// y2 = ff W2 + b2 + xm.
__global__ void t2s_ffn2_kernel(T2sLayer L, const float* __restrict__ ff, const float* __restrict__ xm, float* __restrict__ y2,
                                const int* __restrict__ st, int B, int H, int F);
// logits = h Wp for the utterances about to sample; h = LN2_last(y2) when this step ran the layers, else hx (the prefill's).
__global__ void t2s_logits_kernel(const float* __restrict__ wp, int ldw, const float* __restrict__ lng, const float* __restrict__ lnb,
                                  float eps, const float* __restrict__ y2, const float* __restrict__ hx, float* __restrict__ lg,
                                  const int* __restrict__ st, int B, int H, int V);
// One CTA per utterance: advances NY, then (when due) penalty, top-p, temperature, top-k, softmax, argmax(probs / q), append,
// stop tests.  q: caller rows [B][q_ld][V] or null (Philox); raw: [B][logits_ld][V] raw logits of every sampled step, or null.
__global__ void t2s_sample_kernel(const float* __restrict__ lg, const T2sPrm* __restrict__ prm, const unsigned long long* __restrict__ seeds,
                                  const float* __restrict__ q, float* __restrict__ raw, int* __restrict__ st, int* __restrict__ y,
                                  unsigned* __restrict__ seen, int* __restrict__ n_stopped, int V);

}  // namespace vtts
