// resample.cuh -- rational resampling of recordings (scipy.signal.resample_poly's definition, oracle/resample_oracle.py) and the
// frame energies of librosa.effects.trim, for vtts_resample.
//
// Output m of a clip resampled by up / down is y[m] = sum_q h[p + up q] x[j0 - q] with t = m down + half, p = t mod up,
// j0 = t div up, half = 10 max(up, down), x zero outside the clip.  The taps come per phase, [up][K], K = ceil(L / up), zeros
// past L.  fp32 FFMA on purpose: 44.1 -> 16 kHz is 56 MACs per output sample, so the call is bound by memory traffic and
// launches, not by arithmetic, and tensor cores would not shorten it.
#pragma once
#include "kernels.cuh"

namespace vtts {

constexpr int RS_THREADS = 256;
constexpr int RS_TILE_MAX = 1024;                 // outputs of one CTA at most
constexpr int RS_WIN_MAX = 16384;                 // input window of one CTA at most (floats, 64 KB)
constexpr int RS_TAPS_SMEM = 16384;               // taps of every phase go to shared memory up to this many (64 KB)
constexpr int RS_FRAME = 2048, RS_HOP = 512;      // librosa.effects.trim's frame_length, hop_length
constexpr int RS_FRAME_WARPS = 8;

// Input samples CTA of tile `tile` needs: window [j_lo, j_lo + rs_window) with j_lo = (m0 down + half) div up - (K - 1).
__host__ __device__ inline int rs_window(int tile, int up, int down, int K) {
  return (int)(((int64_t)(tile - 1) * down + up - 1) / up) + K + 1;
}

// Row pitch of the taps in shared memory: odd, so that threads on different phases spread over the banks.
__host__ __device__ inline int rs_taps_pitch(int K) { return K | 1; }

// One CTA resamples outputs [m0, m0 + tile) of clip blockIdx.y.  tab: [in_off B][in_len B][out_off B][out_len B] (packed rows).
// The input window goes to shared memory with coalesced loads (zeros outside the clip); the taps too when `taps_smem`, at
// row pitch rs_taps_pitch(K).
// Each output is one FMA chain over its phase's taps in ascending q, so a clip's output does not depend on the tile, the batch
// or its place in it.
__global__ void __launch_bounds__(RS_THREADS)
resample_kernel(const float* __restrict__ x, const int* __restrict__ tab, int B, const float* __restrict__ taps, int up, int down,
                int K, int half, int tile, int taps_smem, float* __restrict__ y) {
  PDL_LAUNCH();
  extern __shared__ __align__(16) float rs_sm[];
  const int b = blockIdx.y;
  const int64_t m0 = (int64_t)blockIdx.x * tile;
  const int tid = threadIdx.x;
  float* hs = rs_sm;
  const int ks = taps_smem ? rs_taps_pitch(K) : K;
  float* xw = rs_sm + (taps_smem ? up * ks : 0);
  if (taps_smem) {                                  // the taps do not depend on the predecessor kernel: loaded before the wait
    for (int i = tid; i < up * K; i += RS_THREADS) hs[i / K * ks + i % K] = taps[i];
  }
  PDL_WAIT();
  const int n = tab[B + b], nout = tab[3 * B + b];
  if (m0 >= nout) return;
  const float* xc = x + tab[b];
  const int64_t j_lo = (m0 * down + half) / up - (K - 1);
  const int win = rs_window(tile, up, down, K);
  for (int i = tid; i < win; i += RS_THREADS) {
    const int64_t j = j_lo + i;
    xw[i] = (j >= 0 && j < n) ? xc[j] : 0.f;
  }
  __syncthreads();
  const float* hb = taps_smem ? hs : taps;
  const int64_t m_end = min(m0 + tile, (int64_t)nout);
  float* yc = y + tab[2 * B + b];
  for (int64_t m = m0 + tid; m < m_end; m += RS_THREADS) {
    const int64_t t = m * down + half;
    const int p = (int)(t % up);
    const float* hp = hb + p * ks;
    const float* xp = xw + (t / up - j_lo);
    float acc = 0.f;
    for (int q = 0; q < K; ++q) acc = fmaf(hp[q], xp[-q], acc);
    yc[m] = acc;
  }
}

// Sum of squares of every centred frame of every clip in fp64: frame f of clip b covers y[512 f - 1024, 512 f + 1024) (zeros
// outside the clip), 1 + len / 512 frames.  tab: [y_off B][y_len B][e_off B].  One warp per frame; lane l sums samples l,
// l + 32, ... in order, then a fixed butterfly: the energies are the same alone and in any batch.
__global__ void __launch_bounds__(RS_FRAME_WARPS * 32)
frame_energy_kernel(const float* __restrict__ y, const int* __restrict__ tab, int B, double* __restrict__ e) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y;
  const int f = blockIdx.x * RS_FRAME_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n = tab[B + b];
  if (f > n / RS_HOP) return;
  const float* yc = y + tab[b];
  const int a = f * RS_HOP - RS_FRAME / 2;
  double s = 0.0;
  for (int i = lane; i < RS_FRAME; i += 32) {
    const int j = a + i;
    if (j >= 0 && j < n) {
      const double v = (double)yc[j];
      s = fma(v, v, s);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) e[tab[2 * B + b] + f] = s;
}

}  // namespace vtts
