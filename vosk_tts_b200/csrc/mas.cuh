// mas.cuh -- Monotonic Alignment Search on the GPU (the reference runs it on the host: the score matrix is copied to the
// CPU, a Cython loop per batch item under prange, and the path is copied back -- training/vits2/monotonic_align/
// __init__.py:6-22, core.pyx:7-43).  Same recurrence, same evaluation order per cell, fp32 adds only => bit-identical paths.
//
//   forward (core.pyx:16-29):  value[y, x] += max(value[y-1, x-1], value[y-1, x])   for max(0, t_x + y - t_y) <= x < min(t_x, y + 1)
//                              with value[-1, -1] := 0, everything else outside the band := -1e9
//   backtrack (core.pyx:31-34): index = t_x - 1; for y = t_y-1 .. 0: path[y, index] = 1;
//                              if index != 0 and (index == y or value[y-1, index] < value[y-1, index-1]): index -= 1
//
// One CTA per batch item; a row of the band is computed by all threads in parallel (each cell depends on two cells of the
// previous row only), the previous row is kept in shared memory (ping-pong), the raw scores of the next row are prefetched
// into registers before the row barrier.  HBM-bound integer/float work: T_y * T_x * 4 bytes read + written once, plus the
// path (zero-filled by the caller's memset, T_y ones written).  The backtrack is a dependent chain of T_y steps of one thread.
//
// The engine's forced alignment (vtts_align) computes the scores on the device with neg_cent_kernel and asks mas_kernel for
// compact outputs instead of the dense path: the token of every frame, the frames of every token and the path score.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "kernels.cuh"

namespace vtts {

constexpr int MAS_THREADS = 256;
constexpr int MAS_MAXPT = 8;        // columns per thread: T_x <= MAS_THREADS * MAS_MAXPT

// Optional compact outputs, written by thread 0 in the backtrack (each pointer may be null; all null with a path is the
// reference's interface):  token_of_frame[tof_off[b] + y] (tof_off null: b * Ty + y) = the token frame y is aligned to;
// durations[dur_off[b] + x] (dur_off null: b * Tx + x) = the frames of token x (the reference's w = attn.sum(2));
// score[b] = value[t_y - 1][t_x - 1], the log-likelihood of the best path.  path may be null (no dense output, no memset).
__global__ void __launch_bounds__(MAS_THREADS)
mas_kernel(float* __restrict__ value, int* __restrict__ path, const int* __restrict__ t_ys, const int* __restrict__ t_xs, int Ty, int Tx,
           int* __restrict__ token_of_frame, const int* __restrict__ tof_off, int* __restrict__ durations,
           const int* __restrict__ dur_off, float* __restrict__ score) {
  PDL_LAUNCH();
  PDL_WAIT();                                     // value and the lengths may come from the preceding kernels
  extern __shared__ float mas_rows[];            // [2][Tx]
  const int b = blockIdx.x;
  float* v = value + (size_t)b * Ty * Tx;
  int* p = path ? path + (size_t)b * Ty * Tx : nullptr;
  const int t_y = min(t_ys[b], Ty), t_x = min(t_xs[b], Tx);
  if (t_y <= 0 || t_x <= 0) return;
  const float MAXNEG = -1e9f;
  const int tid = threadIdx.x;
  float raw[MAS_MAXPT];                           // scores of the row about to be processed, columns tid + k * MAS_THREADS
#pragma unroll
  for (int k = 0; k < MAS_MAXPT; ++k) {
    const int x = tid + k * MAS_THREADS;
    raw[k] = x < t_x ? v[x] : 0.f;
  }
  for (int y = 0; y < t_y; ++y) {
    float* cur = mas_rows + (y & 1) * Tx;
    const float* prv = mas_rows + ((y & 1) ^ 1) * Tx;
    const int lo = max(0, t_x + y - t_y), hi = min(t_x, y + 1);
    float nxt[MAS_MAXPT];
#pragma unroll
    for (int k = 0; k < MAS_MAXPT; ++k) {         // prefetch row y + 1 (independent of this row's results)
      const int x = tid + k * MAS_THREADS;
      nxt[k] = (x < t_x && y + 1 < t_y) ? v[(size_t)(y + 1) * Tx + x] : 0.f;
    }
#pragma unroll
    for (int k = 0; k < MAS_MAXPT; ++k) {
      const int x = tid + k * MAS_THREADS;
      if (x >= lo && x < hi) {
        const float v_cur = (x == y) ? MAXNEG : prv[x];
        const float v_prev = (x == 0) ? (y == 0 ? 0.f : MAXNEG) : prv[x - 1];
        const float nv = __fadd_rn(raw[k], v_prev > v_cur ? v_prev : v_cur);
        v[(size_t)y * Tx + x] = nv;
        cur[x] = nv;
      }
    }
#pragma unroll
    for (int k = 0; k < MAS_MAXPT; ++k) raw[k] = nxt[k];
    __syncthreads();                              // row y complete (shared + this CTA's global writes) before row y + 1 reads it
  }
  if (tid == 0) {
    int* tof = token_of_frame ? token_of_frame + (tof_off ? (size_t)tof_off[b] : (size_t)b * Ty) : nullptr;
    int* dur = durations ? durations + (dur_off ? (size_t)dur_off[b] : (size_t)b * Tx) : nullptr;
    if (score) score[b] = v[(size_t)(t_y - 1) * Tx + t_x - 1];
    int index = t_x - 1, run = 0;
    for (int y = t_y - 1; y >= 0; --y) {
      if (p) p[(size_t)y * Tx + index] = 1;
      if (tof) tof[y] = index;
      ++run;
      if (index != 0 && (index == y || v[(size_t)(y - 1) * Tx + index] < v[(size_t)(y - 1) * Tx + index - 1])) {
        if (dur) dur[index] = run;              // the path leaves token `index` for good: every token is visited (monotonic,
        run = 0;                                //   one step at most, ending at token 0), so no memset is needed
        --index;
      }
    }
    if (dur) dur[0] = run;
  }
}

// ------------------------------------------------------------------------------------------------
// Gaussian log-likelihood of every frame under every token's prior (SynthesizerTrn.forward, models.py:1645-1651), in the
// DIRECT form
//   neg_cent[b][j][i] = sum_d [ -0.5 log 2pi - logs_p[i,d] - 0.5 (z_p[j,d] - m_p[i,d])^2 exp(-2 logs_p[i,d]) ]
// for frames j < t_y[b], tokens i < t_x[b] (the full rectangle; nothing else is written).  The reference expands the square
// into three GEMM-shaped terms whose rounding error scales with their sum -- largest where z ~ m, i.e. on the path MAS picks,
// and MAS is an argmax.  Here each (j, i, d) is one subtract, one multiply and one FMA in fp32, every precision mode.
// Operands: z rows [frm_off[b] + j][I] (channels-last frames), stats rows [tok_off[b] + i][2I] = [m | logs] of the text
// encoder.  One CTA = NC_T frames x NC_T tokens of one utterance; per chunk of NC_D channels both operands are staged in
// shared memory, with s = -0.5 exp(-2 logs) computed once per (token, channel) of the tile.  The per-token constant
// c[i] = sum_d (-0.5 log 2pi - logs[i,d]) is summed in channel order by one thread per token from the staged chunks, and added
// last.  Output: out[b][Ty][Tx].
// ------------------------------------------------------------------------------------------------
constexpr int NC_T = 32, NC_D = 32, NC_THREADS = 256;

__global__ void __launch_bounds__(NC_THREADS)
neg_cent_kernel(const float* __restrict__ z, const float* __restrict__ stats, int I, const int* __restrict__ frm_len,
                const int* __restrict__ frm_off, const int* __restrict__ tok_len, const int* __restrict__ tok_off,
                float* __restrict__ out, int Ty, int Tx) {
  __shared__ float zs[NC_T][NC_D + 1];
  __shared__ float ms[NC_T][NC_D + 1];
  __shared__ float ss[NC_T][NC_D + 1];
  __shared__ float ls[NC_T][NC_D + 1];
  __shared__ float cs[NC_T];
  const int b = blockIdx.z, i0 = blockIdx.x * NC_T, j0 = blockIdx.y * NC_T;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const float HALF_LOG_2PI = 0.91893853320467274178f;
  PDL_LAUNCH();
  PDL_WAIT();                                      // z and stats come from the preceding kernels
  const int t_y = min(frm_len[b], Ty), t_x = min(tok_len[b], Tx);
  if (i0 >= t_x || j0 >= t_y) return;
  const long zr = (long)frm_off[b] + j0, sr = (long)tok_off[b] + i0;
  const int nj = min(NC_T, t_y - j0), ni = min(NC_T, t_x - i0);
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  float c = 0.f;                                   // c[i0 + tid], threads tid < NC_T
  for (int d0 = 0; d0 < I; d0 += NC_D) {
    for (int e = tid; e < NC_T * NC_D; e += NC_THREADS) {
      const int r = e / NC_D, d = e % NC_D, dd = d0 + d;
      const bool in_d = dd < I;
      zs[r][d] = (r < nj && in_d) ? z[(zr + r) * I + dd] : 0.f;
      const float* srow = stats + (sr + r) * 2 * I;
      const float lg = (r < ni && in_d) ? srow[I + dd] : 0.f;
      ms[r][d] = (r < ni && in_d) ? srow[dd] : 0.f;
      ss[r][d] = (r < ni && in_d) ? -0.5f * expf(-2.f * lg) : 0.f;
      ls[r][d] = lg;
    }
    __syncthreads();
    if (tid < NC_T)
      for (int d = 0; d < NC_D && d0 + d < I; ++d) c = __fsub_rn(__fsub_rn(c, HALF_LOG_2PI), ls[tid][d]);
#pragma unroll 8
    for (int d = 0; d < NC_D; ++d) {
      const float z0 = zs[ty][d], z1 = zs[ty + 16][d];
      const float m0 = ms[tx][d], m1 = ms[tx + 16][d], s0 = ss[tx][d], s1 = ss[tx + 16][d];
      float q;
      q = __fsub_rn(z0, m0); acc[0][0] = fmaf(__fmul_rn(q, s0), q, acc[0][0]);
      q = __fsub_rn(z0, m1); acc[0][1] = fmaf(__fmul_rn(q, s1), q, acc[0][1]);
      q = __fsub_rn(z1, m0); acc[1][0] = fmaf(__fmul_rn(q, s0), q, acc[1][0]);
      q = __fsub_rn(z1, m1); acc[1][1] = fmaf(__fmul_rn(q, s1), q, acc[1][1]);
    }
    __syncthreads();
  }
  if (tid < NC_T) cs[tid] = c;
  __syncthreads();
  float* o = out + (size_t)b * Ty * Tx;
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int j = ty + 16 * a, i = tx + 16 * c;
      if (j < nj && i < ni) o[(size_t)(j0 + j) * Tx + i0 + i] = __fadd_rn(cs[i], acc[a][c]);
    }
}

}  // namespace vtts
