// sovits.cuh -- the kernel of GPT-SoVITS's SynthesizerTrn.extract_latent (module/models.py:990-993) that the dense conv kernel
// does not cover: the codebook argmax of EuclideanCodebook.quantize (module/core_vq.py:175-183).  ssl_proj and the scores
// 2 x.E - |E|^2 (the reference's -|x - E|^2 without the row constant |x|^2) are conv_kernel launches; this picks the best code
// of every score row.  fp32 throughout.
#pragma once
#include "kernels.cuh"

namespace vtts {

constexpr int SVA_WARPS = 8;       // score rows per CTA (one warp each)

// codes[offs[b] + t] = argmax_k s[(offs[b] + t) * K + k] for t < lens[b], the lowest index among equal scores (torch.max's
// index on ties).  Each row is reduced by one warp in a fixed order, whatever the batch and the grid.  grid (row blocks, B).
__global__ void __launch_bounds__(32 * SVA_WARPS)
sv_argmax_kernel(const float* __restrict__ s, int K, const int* __restrict__ lens, const int* __restrict__ offs, int* __restrict__ codes) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const int t = blockIdx.x * SVA_WARPS + (threadIdx.x >> 5);
  if (t >= lens[b]) return;                          // (uniform over the warp)
  const long r = (long)offs[b] + t;
  const float* row = s + r * K;
  float best = -INFINITY;
  int bi = K;                                        // K: no finite score seen
  for (int k = lane; k < K; k += 32) {
    const float v = row[k];
    if (v > best) { best = v; bi = k; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) codes[r] = bi < K ? bi : 0;
}

}  // namespace vtts
