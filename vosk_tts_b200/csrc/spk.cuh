// spk.cuh -- the speaker encoder of QuickVC (SpeakerEncoder, vc/models.py:728-767): a 3-layer LSTM (80 -> 256) over
// 128-frame slices of the target's log-mel, linear 256 -> 256, ReLU, L2 normalisation and the mean over a clip's slices.
//
// The input projection W_ih x + b_ih + b_hh of every layer is a 1x1 conv on the FFMA conv kernel (kernels.cuh).  What is
// left is the recurrence h_t = cell(xp_t + W_hh h_{t-1}): 128 dependent steps per layer.  One thread-block cluster of
// SPK_CTAS CTAs runs NS sequences: CTA r keeps the gate rows of hidden units [32 r, 32 r + 32) of W_hh (4 gates x 32 units x
// 256 = 128 KB) resident in shared memory for the whole sequence, computes those rows for every sequence from h_{t-1} in
// its own shared memory, applies the cell (PyTorch gate order i, f, g, o) and pushes its 32 values of h_t into every CTA's
// next h buffer over DSMEM.  One cluster barrier per step separates the steps; h is double buffered, so a CTA that runs
// ahead writes the buffer nobody reads in that step.  fp32 FFMA in every precision mode.
#pragma once
#include <cooperative_groups.h>
#include "kernels.cuh"

namespace vtts {

constexpr int SPK_H = 256;                        // hidden = embedding = gin_channels (models.py:728, SpeakerEncoder defaults)
constexpr int SPK_GATES = 4 * SPK_H;              // rows of W_ih / W_hh
constexpr int SPK_CTAS = 8;                       // CTAs of one cluster
constexpr int SPK_U = SPK_H / SPK_CTAS;           // hidden units per CTA (32)
constexpr int SPK_THREADS = 256;
constexpr int SPK_WARPS = SPK_THREADS / 32;
constexpr int SPK_KW = SPK_H / SPK_WARPS;         // k range of one warp's partial mat-vec (32)
constexpr int SPK_SLICE = 128, SPK_HOP = 64;      // embed_utterance(partial_frames=128, partial_hop=64), models.py:750

template <int NS>
constexpr size_t spk_rec_smem() {
  return (size_t)(SPK_H * 4 * SPK_U + 2 * NS * SPK_H + SPK_WARPS * NS * 4 * SPK_U) * sizeof(float);
}

__device__ __forceinline__ float spk_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// One LSTM layer over nseq sequences.  Sequence s reads its projected inputs from rows xrow[s] + t of xp ([rows][1024], gate
// order i, f, g, o) and writes h_t to rows orow[s] + t of hout ([rows][256]) for t < len[s]; h_{-1} = c_{-1} = 0.
// whh: W_hh of the layer in the CTA-blocked layout of weights.pack_quickvc: [rank][k][gate * 32 + unit], so that CTA r copies
// one contiguous 128 KB block and lane u of a warp reads unit u of a gate row with consecutive addresses.
// Grid: ceil(nseq / NS) clusters of SPK_CTAS CTAs; cluster q runs sequences [q NS, q NS + NS).
template <int NS>
__global__ void __cluster_dims__(SPK_CTAS, 1, 1) __launch_bounds__(SPK_THREADS, 1)
lstm_rec_kernel(const float* __restrict__ xp, const float* __restrict__ whh, const int* __restrict__ xrow,
                const int* __restrict__ len, const int* __restrict__ orow, int nseq, float* __restrict__ hout) {
  PDL_LAUNCH();
  namespace cg = cooperative_groups;
  cg::cluster_group cl = cg::this_cluster();
  extern __shared__ __align__(16) float sm[];
  float* W = sm;                                   // [SPK_H k][4 * SPK_U]
  float* hb = W + SPK_H * 4 * SPK_U;               // [2][NS][SPK_H]
  float* part = hb + 2 * NS * SPK_H;               // [SPK_WARPS][NS][4 * SPK_U]
  const int rank = (int)cl.block_rank();
  const int s0 = (blockIdx.x / SPK_CTAS) * NS;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  {   // the weights do not depend on the predecessor kernel: loaded before the wait
    const float4* src = reinterpret_cast<const float4*>(whh + (size_t)rank * SPK_H * 4 * SPK_U);
    float4* dst = reinterpret_cast<float4*>(W);
    for (int i = tid; i < SPK_H * SPK_U; i += SPK_THREADS) dst[i] = src[i];
    for (int i = tid; i < NS * SPK_H; i += SPK_THREADS) hb[i] = 0.f;
  }
  PDL_WAIT();
  // thread tid < NS * SPK_U owns the cell of (sequence cs, unit cj) for the whole sequence: c stays in a register
  const bool cell = tid < NS * SPK_U;
  const int cs = tid / SPK_U, cj = tid % SPK_U;
  int xr = 0, L = 0, orw = 0;
  if (cell && s0 + cs < nseq) { xr = xrow[s0 + cs]; L = len[s0 + cs]; orw = orow[s0 + cs]; }
  int T = 0;
  for (int s = 0; s < NS && s0 + s < nseq; ++s) T = max(T, len[s0 + s]);
  float c = 0.f;
  cl.sync();                                       // every CTA's h_{-1} is zero before anyone pushes h_0 into it
  for (int t = 0; t < T; ++t) {
    const float* hc = hb + (t & 1) * NS * SPK_H;
    const bool act = t < L;
    float xg[4] = {0.f, 0.f, 0.f, 0.f};
    if (act) {                                     // issued before the mat-vec, which hides its latency
      const float* x = xp + (size_t)(xr + t) * SPK_GATES + rank * SPK_U + cj;
#pragma unroll
      for (int g = 0; g < 4; ++g) xg[g] = x[g * SPK_H];
    }
    float acc[NS][4];
#pragma unroll
    for (int s = 0; s < NS; ++s)
#pragma unroll
      for (int g = 0; g < 4; ++g) acc[s][g] = 0.f;
    const int k0 = warp * SPK_KW;
#pragma unroll 2
    for (int kk = 0; kk < SPK_KW; kk += 4) {
      float w[4][4];
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int g = 0; g < 4; ++g) w[q][g] = W[(k0 + kk + q) * 4 * SPK_U + g * SPK_U + lane];
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        const float4 hv = *reinterpret_cast<const float4*>(hc + s * SPK_H + k0 + kk);
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          float a = acc[s][g];
          a = fmaf(w[0][g], hv.x, a);
          a = fmaf(w[1][g], hv.y, a);
          a = fmaf(w[2][g], hv.z, a);
          a = fmaf(w[3][g], hv.w, a);
          acc[s][g] = a;
        }
      }
    }
#pragma unroll
    for (int s = 0; s < NS; ++s)
#pragma unroll
      for (int g = 0; g < 4; ++g) part[(warp * NS + s) * 4 * SPK_U + g * SPK_U + lane] = acc[s][g];
    __syncthreads();
    if (cell && act) {
      float pre[4];
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        float a = xg[g];
#pragma unroll
        for (int w8 = 0; w8 < SPK_WARPS; ++w8) a += part[(w8 * NS + cs) * 4 * SPK_U + g * SPK_U + cj];
        pre[g] = a;
      }
      const float ig = spk_sigmoid(pre[0]), fg = spk_sigmoid(pre[1]), gg = tanhf(pre[2]), og = spk_sigmoid(pre[3]);
      c = fmaf(fg, c, ig * gg);
      const float h = og * tanhf(c);
      hout[(size_t)(orw + t) * SPK_H + rank * SPK_U + cj] = h;
      float* dst = hb + ((t + 1) & 1) * NS * SPK_H + cs * SPK_H + rank * SPK_U + cj;
#pragma unroll
      for (int r = 0; r < SPK_CTAS; ++r) *cl.map_shared_rank(dst, r) = h;
    }
    cl.sync();                                     // h_t complete in every CTA; part and h_{t-1} free again
  }
}

// g[b] = mean over the slices s of clip b (seq_of_clip[b] <= s < seq_of_clip[b + 1], in that order) of
// e_s / ||e_s||,  e_s = relu(W h_s + bias), h_s = row last[s] of h (the last layer's final hidden state, hidden[-1]).
// lin_w: [SPK_H k][SPK_H out] (nn.Linear weight transposed).  One CTA per clip, one thread per output.
__global__ void __launch_bounds__(SPK_H)
spk_embed_kernel(const float* __restrict__ h, const int* __restrict__ last, const int* __restrict__ seq_of_clip,
                 const float* __restrict__ lin_w, const float* __restrict__ lin_b, float* __restrict__ g) {
  PDL_LAUNCH();
  PDL_WAIT();
  __shared__ float hs[SPK_H];
  __shared__ float red[SPK_H / 32];
  const int b = blockIdx.x, o = threadIdx.x, warp = o >> 5, lane = o & 31;
  const int s_begin = seq_of_clip[b], s_end = seq_of_clip[b + 1];
  float sum = 0.f;
  for (int s = s_begin; s < s_end; ++s) {
    __syncthreads();
    hs[o] = h[(size_t)last[s] * SPK_H + o];
    __syncthreads();
    float a = lin_b[o];
    for (int k = 0; k < SPK_H; ++k) a = fmaf(lin_w[k * SPK_H + o], hs[k], a);
    a = fmaxf(a, 0.f);
    float q = a * a;
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) q += __shfl_xor_sync(0xffffffffu, q, m);
    if (lane == 0) red[warp] = q;
    __syncthreads();
    float n2 = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < SPK_H / 32; ++w8) n2 += red[w8];
    sum += a / sqrtf(n2);
  }
  g[(size_t)b * SPK_H + o] = sum / (float)(s_end - s_begin);
}

}  // namespace vtts
