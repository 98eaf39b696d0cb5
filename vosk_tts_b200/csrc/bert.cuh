// bert.cuh -- the embedding stage of BERT (transformers' BertEmbeddings, as training/stabletts/matcha/onnx/bert-export.py
// exports it): word + token-type 0 + absolute position embeddings, then LayerNorm.  The encoder layers after it are the
// post-LN transformer ContentVec runs (engine.cu post_ln_layers).  fp32 FFMA.
#pragma once
#include "kernels.cuh"
#include "contentvec.cuh"

namespace vtts {

// One warp per word piece: row offs[b] + t of sentence b gets LN(word[ids[row]] + pos[t] + type0), positions counted from
// the sentence's own start (each sentence is embedded as if alone).  p_hi / p_lo (or null): the split-bf16 planes of the
// output rows, the operand of the first qkv GEMM on the tensor cores.  grid (ceil(maxLen / CVL_WARPS), B).
__global__ void __launch_bounds__(32 * CVL_WARPS)
bert_embed_kernel(const int* __restrict__ ids, const float* __restrict__ word, const float* __restrict__ pos, const float* __restrict__ type0,
                  const float* __restrict__ g, const float* __restrict__ bt, float eps, float* __restrict__ out, const int* __restrict__ lens,
                  const int* __restrict__ offs, int C, __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * CVL_WARPS + warp;
  if (t >= lens[b]) return;
  const long row = (long)offs[b] + t;
  const float* wr = word + (long)ids[row] * C;
  const float* pr = pos + (long)t * C;
  float v[CVL_MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < CVL_MAXV; ++i) {
    const int c = lane + 32 * i;
    float u = 0.f;
    if (c < C) u = (wr[c] + type0[c]) + pr[c];   // the order of BertEmbeddings: (inputs + token_type) + position
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
      out[row * C + c] = o;
      if (p_hi) split_bf16(o, p_hi[row * C + c], p_lo[row * C + c]);
    }
  }
}

}  // namespace vtts
