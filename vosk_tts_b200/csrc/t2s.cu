// t2s.cu -- GPT-SoVITS text-to-semantic decoding: the kernels declared in t2s.cuh (see there and DESIGN.md 4.s).
//
// A translation unit of its own (as st_gather.cu and st_tc.cu) so that engine.cu's module, which ptxas compiles as a whole,
// holds exactly the kernels it held before: every existing kernel keeps its machine code bit for bit.  These kernels do not
// stamp vtts_timeline (g_timeline lives in engine.cu's module).
//
// Every kernel waits for its predecessor before it reads anything, then lets its successor launch (the PDL order of
// kernels.cuh's PDL_WAIT).  Each decode GEMV gives one output column to one lane and a fixed slice of the input width to
// each of its T2S_WARPS warps, and sums the partial dot products in warp order: an utterance's rows are computed by the same operations
// in the same order whatever the batch and whichever row tile holds them.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <math.h>
#include <stdint.h>

#include "t2s.cuh"

namespace vtts {

#define T2S_PDL() asm volatile("griddepcontrol.wait;\n\tgriddepcontrol.launch_dependents;" ::: "memory")

namespace {

// The split-bf16 operand planes of the tensor-core GEMMs (kernels.cuh split_bf16: hi = rne(x), lo = rne(x - hi)).
__device__ __forceinline__ void t2s_split(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  const uint32_t h = (__float_as_uint(x) + 0x8000u) & 0xFFFF0000u;
  const float r = x - __uint_as_float(h);
  const uint32_t l = __float_as_uint(r) + 0x8000u;
  hi = __ushort_as_bfloat16((unsigned short)(h >> 16));
  lo = __ushort_as_bfloat16((unsigned short)(l >> 16));
}

__device__ __forceinline__ bool runs_layers(const int* s) { return !s[ST_STOP] && s[ST_NY] < s[ST_P] + s[ST_GEN]; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// LayerNorm of one row by one warp (torch.nn.LayerNorm: biased variance, (x - mean) * rstd * g + b), into dst.
__device__ __forceinline__ void warp_ln(const float* __restrict__ src, const float* __restrict__ g, const float* __restrict__ bt, float eps,
                                        float* dst, int H) {
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int c = lane; c < H; c += 32) {
    const float v = src[c];
    dst[c] = v;
    s += v;
  }
  const float mean = warp_sum(s) / (float)H;
  float q = 0.f;
  for (int c = lane; c < H; c += 32) {
    const float d = dst[c] - mean;
    q = fmaf(d, d, q);
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)H + eps);
  for (int c = lane; c < H; c += 32) dst[c] = fmaf((dst[c] - mean) * rstd, g[c], bt[c]);
}

// acc[r] = sum_k xs[r][k] W[k][c] for the T2S_RB rows of the tile; warp w sums k in [w Cin / W, (w + 1) Cin / W) (W =
// T2S_WARPS), 16 weight loads in flight per lane, then warp 0 adds the partials in warp order.  Every thread calls it; the
// result is valid in warp 0.  Cin % T2S_WARPS == 0.
__device__ __forceinline__ void gemv_tile(const float* xs, int Cin, const float* __restrict__ W, int ldw, int c, bool cok,
                                          float (&acc)[T2S_RB], float* red) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kper = Cin / T2S_WARPS, k0 = warp * kper;
#pragma unroll
  for (int r = 0; r < T2S_RB; ++r) acc[r] = 0.f;
  const float* wp = W + (long)k0 * ldw + (cok ? c : 0);
  int k = 0;
  for (; k + 16 <= kper; k += 16) {
    float w[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) w[i] = cok ? __ldg(wp + (long)(k + i) * ldw) : 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
      for (int r = 0; r < T2S_RB; ++r) acc[r] = fmaf(xs[r * Cin + k0 + k + i], w[i], acc[r]);
  }
  for (; k < kper; ++k) {
    const float w = cok ? __ldg(wp + (long)k * ldw) : 0.f;
#pragma unroll
    for (int r = 0; r < T2S_RB; ++r) acc[r] = fmaf(xs[r * Cin + k0 + k], w, acc[r]);
  }
#pragma unroll
  for (int r = 0; r < T2S_RB; ++r) red[(warp * T2S_RB + r) * 32 + lane] = acc[r];
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int r = 0; r < T2S_RB; ++r) {
      float s = 0.f;
      for (int w = 0; w < T2S_WARPS; ++w) s += red[(w * T2S_RB + r) * 32 + lane];
      acc[r] = s;
    }
  }
}

// The rows of this CTA's tile whose layers run this step; false when none does.
__device__ __forceinline__ bool tile_rows(const int* __restrict__ st, int B, bool (&act)[T2S_RB]) {
  bool any = false;
#pragma unroll
  for (int r = 0; r < T2S_RB; ++r) {
    const int b = blockIdx.y * T2S_RB + r;
    act[r] = b < B && runs_layers(st + b * T2S_ST);
    any |= act[r];
  }
  return any;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------
// prefill
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
t2s_prefill_embed_kernel(const int* __restrict__ ids, const float* __restrict__ temb, const float* __restrict__ aemb,
                         const float* __restrict__ bp, const float* __restrict__ bp_bias, const float* __restrict__ pe, float alpha_t,
                         float alpha_a, int H, float* __restrict__ x, const int* __restrict__ lens, const int* __restrict__ offs,
                         const int* __restrict__ init, __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo) {
  T2S_PDL();
  const int b = blockIdx.y, t = blockIdx.x, T = init[b * 4];
  if (t >= lens[b]) return;
  const long row = (long)offs[b] + t;
  if (t < T) {
    const float* er = temb + (long)ids[row] * H;
    for (int c = threadIdx.x; c < H; c += blockDim.x) {
      // infer_panel's order: (ar_text_embedding(x) + bert_proj(bert)) * 1 + alpha * pe, each op rounded on its own
      const float v = __fadd_rn(__fadd_rn(er[c], bp ? bp[row * H + c] : bp_bias[c]), __fmul_rn(alpha_t, pe[(long)t * H + c]));
      x[row * H + c] = v;
      if (p_hi) t2s_split(v, p_hi[row * H + c], p_lo[row * H + c]);
    }
  } else {
    const float* er = aemb + (long)ids[row] * H;      // prompt token j = t - T at audio position j
    for (int c = threadIdx.x; c < H; c += blockDim.x) {
      const float v = __fadd_rn(er[c], __fmul_rn(alpha_a, pe[(long)(t - T) * H + c]));
      x[row * H + c] = v;
      if (p_hi) t2s_split(v, p_hi[row * H + c], p_lo[row * H + c]);
    }
  }
}

// One warp per (row, head): softmax(q k^T / sqrt(dk)) v over the keys row t may see, k < T or k <= t, online over chunks of
// 32 keys in key order (the order does not depend on the batch).
__global__ void __launch_bounds__(32)
t2s_prefix_attn_kernel(const float* __restrict__ qkv, int H, int dk, float scale, float* __restrict__ ao, const int* __restrict__ lens,
                       const int* __restrict__ offs, const int* __restrict__ init, __nv_bfloat16* __restrict__ p_hi,
                       __nv_bfloat16* __restrict__ p_lo) {
  __shared__ __align__(16) float qs[128];
  T2S_PDL();
  const int b = blockIdx.z, h = blockIdx.y, t = blockIdx.x, lane = threadIdx.x;
  if (t >= lens[b]) return;
  const int T = init[b * 4], n = t < T ? T : t + 1;
  const long r0 = offs[b];
  for (int d = lane; d < dk; d += 32) qs[d] = qkv[(r0 + t) * 3 * H + h * dk + d] * scale;
  __syncwarp();
  float m = -INFINITY, l = 0.f, acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int k0 = 0; k0 < n; k0 += 32) {
    const int key = k0 + lane;
    float sc = -INFINITY;
    if (key < n) {
      const float4* kr = reinterpret_cast<const float4*>(qkv + (r0 + key) * 3 * H + H + h * dk);
      sc = 0.f;
      for (int d4 = 0; d4 < dk / 4; ++d4) {
        const float4 k4 = kr[d4];
        sc = fmaf(qs[4 * d4], k4.x, sc);
        sc = fmaf(qs[4 * d4 + 1], k4.y, sc);
        sc = fmaf(qs[4 * d4 + 2], k4.z, sc);
        sc = fmaf(qs[4 * d4 + 3], k4.w, sc);
      }
    }
    const float mn = fmaxf(m, warp_max(sc));
    const float corr = expf(m - mn);
    const float p = key < n ? expf(sc - mn) : 0.f;
    l = fmaf(l, corr, warp_sum(p));
    for (int i = 0; i < dk / 32; ++i) acc[i] *= corr;
    const int cnt = min(32, n - k0);
    for (int j = 0; j < cnt; ++j) {
      const float pj = __shfl_sync(0xffffffffu, p, j);
      const float* vr = qkv + (r0 + k0 + j) * 3 * H + 2 * H + h * dk;
      for (int i = 0; i < dk / 32; ++i) acc[i] = fmaf(pj, vr[i * 32 + lane], acc[i]);
    }
    m = mn;
  }
  for (int i = 0; i < dk / 32; ++i) {
    const long o = (r0 + t) * H + h * dk + i * 32 + lane;
    const float v = acc[i] / l;
    ao[o] = v;
    if (p_hi) t2s_split(v, p_hi[o], p_lo[o]);
  }
}

__global__ void __launch_bounds__(256)
t2s_relu_kernel(float* __restrict__ y, int C, const int* __restrict__ lens, const int* __restrict__ offs, __nv_bfloat16* __restrict__ p_hi,
                __nv_bfloat16* __restrict__ p_lo) {
  T2S_PDL();
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= lens[b]) return;
  const long r = ((long)offs[b] + t) * C;
  for (int c = threadIdx.x; c < C; c += 256) {
    const float v = fmaxf(y[r + c], 0.f);
    if (p_hi) t2s_split(v, p_hi[r + c], p_lo[r + c]);
    else y[r + c] = v;
  }
}

__global__ void __launch_bounds__(128)
t2s_kv_store_kernel(const float* __restrict__ qkv, int H, float* __restrict__ kc, float* __restrict__ vc, const int* __restrict__ lens,
                    const int* __restrict__ offs, const int* __restrict__ init) {
  T2S_PDL();
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= lens[b]) return;
  const float* src = qkv + ((long)offs[b] + t) * 3 * H;
  const long dst = ((long)init[b * 4 + 2] + t) * H;
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    kc[dst + c] = src[H + c];
    vc[dst + c] = src[2 * H + c];
  }
}

// init [B][4]: T, P, first cache row, first token slot.
__global__ void __launch_bounds__(256)
t2s_init_kernel(const int* __restrict__ init, const int* __restrict__ prompt, const int* __restrict__ poffs, const float* __restrict__ pre,
                const int* __restrict__ offs, int H, int V, int* __restrict__ st, int* __restrict__ y, unsigned* __restrict__ seen,
                float* __restrict__ hx) {
  T2S_PDL();
  const int b = blockIdx.x;
  const int T = init[b * 4], P = init[b * 4 + 1], yoff = init[b * 4 + 3], nw = (V + 31) / 32;
  if (threadIdx.x == 0) {
    int* s = st + b * T2S_ST;
    // the prefill ran the layers on every prompt token: the first step samples
    s[ST_T] = T; s[ST_P] = P; s[ST_KV] = init[b * 4 + 2]; s[ST_NY] = P; s[ST_GEN] = 0; s[ST_STOP] = 0; s[ST_YOFF] = yoff; s[7] = 0;
  }
  for (int i = threadIdx.x; i < nw; i += blockDim.x) seen[(long)b * nw + i] = 0u;
  __syncthreads();
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    const int tok = prompt[poffs[b] + i];
    y[yoff + i] = tok;
    atomicOr(&seen[(long)b * nw + (tok >> 5)], 1u << (tok & 31));
  }
  const float* src = pre + ((long)offs[b] + T + P - 1) * H;
  for (int c = threadIdx.x; c < H; c += blockDim.x) hx[(long)b * H + c] = src[c];
}

// ---------------------------------------------------------------------------------------------------
// decode step
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * T2S_WARPS)
t2s_qkv_kernel(T2sLayer L, const float* __restrict__ lnpg, const float* __restrict__ lnpb, const float* __restrict__ aemb,
               const float* __restrict__ pe, float alpha, const int* __restrict__ y, const float* __restrict__ y2, float* __restrict__ x,
               float* __restrict__ q, const int* __restrict__ st, int B, int H) {
  extern __shared__ __align__(16) float t2s_sm[];
  float *xs = t2s_sm, *red = t2s_sm + T2S_RB * H;
  T2S_PDL();
  bool act[T2S_RB];
  if (!tile_rows(st, B, act)) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < T2S_RB) {
    const int b = blockIdx.y * T2S_RB + warp;
    float* xr = xs + warp * H;
    if (act[warp]) {
      const int* s = st + b * T2S_ST;
      const int ny = s[ST_NY];
      if (!lnpg) {          // ar_audio_embedding(y[ny]) * 1 + alpha * pe[ny]
        const float* er = aemb + (long)y[s[ST_YOFF] + ny] * H;
        for (int c = lane; c < H; c += 32) xr[c] = __fadd_rn(er[c], __fmul_rn(alpha, pe[(long)ny * H + c]));
      } else {
        warp_ln(y2 + (long)b * H, lnpg, lnpb, L.eps, xr, H);
      }
      if (blockIdx.x == 0)
        for (int c = lane; c < H; c += 32) x[(long)b * H + c] = xr[c];
    } else {
      for (int c = lane; c < H; c += 32) xr[c] = 0.f;
    }
  }
  __syncthreads();
  const int c = blockIdx.x * T2S_COLS + lane;
  const bool cok = c < 3 * H;
  float acc[T2S_RB];
  gemv_tile(xs, H, L.wqkv, L.ldqkv, c, cok, acc, red);
  if (warp != 0 || !cok) return;
  const float bias = L.bqkv[c];
#pragma unroll
  for (int r = 0; r < T2S_RB; ++r) {
    if (!act[r]) continue;
    const int b = blockIdx.y * T2S_RB + r;
    const int* s = st + b * T2S_ST;
    const float v = acc[r] + bias;
    if (c < H) {
      q[(long)b * H + c] = v;
    } else {
      const long row = (long)s[ST_KV] + s[ST_T] + s[ST_NY];
      if (c < 2 * H) L.kc[row * H + c - H] = v;
      else L.vc[row * H + c - 2 * H] = v;
    }
  }
}

__global__ void __launch_bounds__(32)
t2s_attn_kernel(const float* __restrict__ q, const float* __restrict__ kc, const float* __restrict__ vc, float* __restrict__ part,
                const int* __restrict__ st, int H, int dk, float scale, int nsplit) {
  __shared__ __align__(16) float qs[128];
  T2S_PDL();
  const int b = blockIdx.z, h = blockIdx.y, sp = blockIdx.x, lane = threadIdx.x;
  const int* s = st + b * T2S_ST;
  if (!runs_layers(s)) return;
  const int n = s[ST_T] + s[ST_NY] + 1;           // every text row, every audio row so far, and this token's
  const int k0 = sp * T2S_KS;
  if (k0 >= n) return;
  const int cnt = min(T2S_KS, n - k0);
  const int heads = H / dk;
  for (int d = lane; d < dk; d += 32) qs[d] = q[(long)b * H + h * dk + d] * scale;   // q * sqrt(1 / dk), as the reference scales it
  __syncwarp();
  const long kb = (long)s[ST_KV] + k0;
  float sc[T2S_KS / 32];
#pragma unroll
  for (int j = 0; j < T2S_KS / 32; ++j) {
    const int key = j * 32 + lane;
    float a = -INFINITY;
    if (key < cnt) {
      const float4* kr = reinterpret_cast<const float4*>(kc + (kb + key) * H + h * dk);
      a = 0.f;
      for (int d4 = 0; d4 < dk / 4; ++d4) {
        const float4 k4 = kr[d4];
        a = fmaf(qs[4 * d4], k4.x, a);
        a = fmaf(qs[4 * d4 + 1], k4.y, a);
        a = fmaf(qs[4 * d4 + 2], k4.z, a);
        a = fmaf(qs[4 * d4 + 3], k4.w, a);
      }
    }
    sc[j] = a;
  }
  float m = -INFINITY;
#pragma unroll
  for (int j = 0; j < T2S_KS / 32; ++j) m = fmaxf(m, sc[j]);
  m = warp_max(m);
  float l = 0.f;
#pragma unroll
  for (int j = 0; j < T2S_KS / 32; ++j) {
    sc[j] = j * 32 + lane < cnt ? expf(sc[j] - m) : 0.f;
    l += sc[j];
  }
  l = warp_sum(l);
  float* out = part + ((long)(b * heads + h) * nsplit + sp) * (dk + 2);
  for (int d0 = 0; d0 < dk; d0 += 32) {
    const int d = d0 + lane;
    float a = 0.f;
#pragma unroll
    for (int j = 0; j < T2S_KS / 32; ++j)
      for (int i = 0; i < 32 && j * 32 + i < cnt; ++i) {
        const float p = __shfl_sync(0xffffffffu, sc[j], i);
        if (d < dk) a = fmaf(p, vc[(kb + j * 32 + i) * H + h * dk + d], a);
      }
    if (d < dk) out[2 + d] = a;
  }
  if (lane == 0) { out[0] = m; out[1] = l; }
}

__global__ void __launch_bounds__(32 * T2S_WARPS)
t2s_o_kernel(T2sLayer L, const float* __restrict__ part, const float* __restrict__ x, float* __restrict__ y1, const int* __restrict__ st,
             int B, int H, int dk, int nsplit) {
  extern __shared__ __align__(16) float t2s_sm[];
  float *xs = t2s_sm, *red = t2s_sm + T2S_RB * H;
  T2S_PDL();
  bool act[T2S_RB];
  if (!tile_rows(st, B, act)) return;
  const int heads = H / dk;
#pragma unroll
  for (int r = 0; r < T2S_RB; ++r) {
    const int b = blockIdx.y * T2S_RB + r;
    const int ns = act[r] ? (st[b * T2S_ST + ST_T] + st[b * T2S_ST + ST_NY] + 1 + T2S_KS - 1) / T2S_KS : 0;
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
      if (!act[r]) { xs[r * H + i] = 0.f; continue; }
      const int h = i / dk, d = i - h * dk;
      const float* p = part + (long)(b * heads + h) * nsplit * (dk + 2);
      float M = -INFINITY;
      for (int k = 0; k < ns; ++k) M = fmaxf(M, p[k * (dk + 2)]);
      float Ls = 0.f, A = 0.f;
      for (int k = 0; k < ns; ++k) {
        const float e = expf(p[k * (dk + 2)] - M);
        Ls = fmaf(p[k * (dk + 2) + 1], e, Ls);
        A = fmaf(p[k * (dk + 2) + 2 + d], e, A);
      }
      xs[r * H + i] = A / Ls;
    }
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, c = blockIdx.x * T2S_COLS + lane;
  const bool cok = c < H;
  float acc[T2S_RB];
  gemv_tile(xs, H, L.wo, L.ldo, c, cok, acc, red);
  if (threadIdx.x >= 32 || !cok) return;
  const float bias = L.bo[c];
#pragma unroll
  for (int r = 0; r < T2S_RB; ++r) {
    if (!act[r]) continue;
    const long b = blockIdx.y * T2S_RB + r;
    y1[b * H + c] = x[b * H + c] + (acc[r] + bias);
  }
}

__global__ void __launch_bounds__(32 * T2S_WARPS)
t2s_ffn1_kernel(T2sLayer L, const float* __restrict__ y1, float* __restrict__ xm, float* __restrict__ ff, const int* __restrict__ st,
                int B, int H, int F) {
  extern __shared__ __align__(16) float t2s_sm[];
  float *xs = t2s_sm, *red = t2s_sm + T2S_RB * H;
  T2S_PDL();
  bool act[T2S_RB];
  if (!tile_rows(st, B, act)) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < T2S_RB) {
    const int b = blockIdx.y * T2S_RB + warp;
    float* xr = xs + warp * H;
    if (act[warp]) {
      warp_ln(y1 + (long)b * H, L.ln1g, L.ln1b, L.eps, xr, H);
      if (blockIdx.x == 0)
        for (int c = lane; c < H; c += 32) xm[(long)b * H + c] = xr[c];
    } else {
      for (int c = lane; c < H; c += 32) xr[c] = 0.f;
    }
  }
  __syncthreads();
  const int c = blockIdx.x * T2S_COLS + lane;
  const bool cok = c < F;
  float acc[T2S_RB];
  gemv_tile(xs, H, L.w1, L.ld1, c, cok, acc, red);
  if (warp != 0 || !cok) return;
  const float bias = L.b1[c];
#pragma unroll
  for (int r = 0; r < T2S_RB; ++r)
    if (act[r]) ff[(long)(blockIdx.y * T2S_RB + r) * F + c] = fmaxf(acc[r] + bias, 0.f);
}

__global__ void __launch_bounds__(32 * T2S_WARPS)
t2s_ffn2_kernel(T2sLayer L, const float* __restrict__ ff, const float* __restrict__ xm, float* __restrict__ y2, const int* __restrict__ st,
                int B, int H, int F) {
  extern __shared__ __align__(16) float t2s_sm[];
  float *xs = t2s_sm, *red = t2s_sm + T2S_RB * F;
  T2S_PDL();
  bool act[T2S_RB];
  if (!tile_rows(st, B, act)) return;
#pragma unroll
  for (int r = 0; r < T2S_RB; ++r) {
    const long b = blockIdx.y * T2S_RB + r;
    for (int i = threadIdx.x; i < F; i += blockDim.x) xs[r * F + i] = act[r] ? ff[b * F + i] : 0.f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, c = blockIdx.x * T2S_COLS + lane;
  const bool cok = c < H;
  float acc[T2S_RB];
  gemv_tile(xs, F, L.w2, L.ld2, c, cok, acc, red);
  if (threadIdx.x >= 32 || !cok) return;
  const float bias = L.b2[c];
#pragma unroll
  for (int r = 0; r < T2S_RB; ++r) {
    if (!act[r]) continue;
    const long b = blockIdx.y * T2S_RB + r;
    y2[b * H + c] = xm[b * H + c] + (acc[r] + bias);
  }
}

__global__ void __launch_bounds__(32 * T2S_WARPS)
t2s_logits_kernel(const float* __restrict__ wp, int ldw, const float* __restrict__ lng, const float* __restrict__ lnb, float eps,
                  const float* __restrict__ y2, const float* __restrict__ hx, float* __restrict__ lg, const int* __restrict__ st, int B,
                  int H, int V) {
  extern __shared__ __align__(16) float t2s_sm[];
  float *xs = t2s_sm, *red = t2s_sm + T2S_RB * H;
  T2S_PDL();
  bool act[T2S_RB], ran[T2S_RB], any = false;
#pragma unroll
  for (int r = 0; r < T2S_RB; ++r) {
    const int b = blockIdx.y * T2S_RB + r;
    act[r] = ran[r] = false;
    if (b >= B) continue;
    const int* s = st + b * T2S_ST;
    if (s[ST_STOP]) continue;
    ran[r] = s[ST_NY] < s[ST_P] + s[ST_GEN];
    act[r] = s[ST_NY] + (ran[r] ? 1 : 0) == s[ST_P] + s[ST_GEN];   // this step samples
    any |= act[r];
  }
  if (!any) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < T2S_RB) {
    const int b = blockIdx.y * T2S_RB + warp;
    float* xr = xs + warp * H;
    if (act[warp] && ran[warp]) warp_ln(y2 + (long)b * H, lng, lnb, eps, xr, H);
    else if (act[warp]) for (int c = lane; c < H; c += 32) xr[c] = hx[(long)b * H + c];
    else for (int c = lane; c < H; c += 32) xr[c] = 0.f;
  }
  __syncthreads();
  const int c = blockIdx.x * T2S_COLS + lane;
  const bool cok = c < V;
  float acc[T2S_RB];
  gemv_tile(xs, H, wp, ldw, c, cok, acc, red);
  if (warp != 0 || !cok) return;
#pragma unroll
  for (int r = 0; r < T2S_RB; ++r)
    if (act[r]) lg[(long)(blockIdx.y * T2S_RB + r) * V + c] = acc[r];
}

// ---------------------------------------------------------------------------------------------------
// sampler (ar/models/utils.py:110-161 with the loop's stop rules, t2s_model.py:395-416)
// ---------------------------------------------------------------------------------------------------
namespace {

__device__ __forceinline__ void philox4x32_t2s(uint32_t (&ctr)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr[0]), lo0 = 0xD2511F53u * ctr[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr[2]), lo1 = 0xCD9E8D57u * ctr[2];
    const uint32_t n0 = hi1 ^ ctr[1] ^ k0, n1 = lo1, n2 = hi0 ^ ctr[3] ^ k1, n3 = lo0;
    ctr[0] = n0; ctr[1] = n1; ctr[2] = n2; ctr[3] = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}

// Exp(1) draw of entry v at sampling step `step`: a Philox stream keyed by (step, v) under the utterance's seed.
__device__ __forceinline__ float philox_exp(uint64_t seed, uint32_t step, uint32_t v) {
  uint32_t ctr[4] = {step, v, 11u, 0x5eedu};
  philox4x32_t2s(ctr, (uint32_t)seed, (uint32_t)(seed >> 32));
  const float u = ((float)(ctr[0] >> 8) + 0.5f) * (1.f / 16777216.f);     // (0, 1)
  return -logf(u);
}

// a sorts before b: larger value first, then smaller index
__device__ __forceinline__ bool before(float av, int ai, float bv, int bi) { return av > bv || (av == bv && ai < bi); }

__device__ float block_sum(float v, float* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sh[w];
  return t;
}

// block argmax over (value, index): the larger value, the smaller index on ties
__device__ void block_argmax(float& v, int& i, float* shv, int* shi) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (before(ov, oi, v, i)) { v = ov; i = oi; }
  }
  __syncthreads();
  if (lane == 0) { shv[warp] = v; shi[warp] = i; }
  __syncthreads();
  v = shv[0]; i = shi[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
    if (before(shv[w], shi[w], v, i)) { v = shv[w]; i = shi[w]; }
}

}  // namespace

__global__ void __launch_bounds__(T2S_SAMPLE_THREADS)
t2s_sample_kernel(const float* __restrict__ lg, const T2sPrm* __restrict__ prm, const unsigned long long* __restrict__ seeds,
                  const float* __restrict__ q, float* __restrict__ raw, int* __restrict__ st, int* __restrict__ y,
                  unsigned* __restrict__ seen, int* __restrict__ n_stopped, int V) {
  __shared__ float kv[T2S_MAX_V];
  __shared__ int ki[T2S_MAX_V];
  __shared__ float shv[32], scan[32];
  __shared__ int shi[32];
  T2S_PDL();
  const int b = blockIdx.x, tid = threadIdx.x;
  int* s = st + b * T2S_ST;
  const int stop0 = s[ST_STOP], P = s[ST_P], gen = s[ST_GEN], yoff = s[ST_YOFF];
  int ny = s[ST_NY];
  if (stop0) return;
  if (ny < P + gen) ++ny;                          // the layers ran on token y[ny] this step
  __syncthreads();
  if (tid == 0) s[ST_NY] = ny;
  if (ny != P + gen) return;                       // (the prefill has run the layers on the whole prompt)
  const T2sPrm pr = *prm;
  const int Vv = gen == 0 ? V - 1 : V;             // step 0 drops the EOS column (logits[:, :-1])
  int NS = 1;
  while (NS < Vv) NS <<= 1;
  const unsigned* sn = seen + (long)b * ((V + 31) / 32);
  // repetition penalty on every token of y (prompt included), in place: the EOS test below sees the penalised logits
  float pv = -INFINITY;
  int pi = 0x7fffffff;
  for (int v = tid; v < NS; v += blockDim.x) {
    float l = -INFINITY;
    if (v < Vv) {
      l = lg[(long)b * V + v];
      if (raw && gen < pr.logits_ld) raw[((long)b * pr.logits_ld + gen) * V + v] = l;
      if ((sn[v >> 5] >> (v & 31)) & 1u) l = l < 0.f ? __fmul_rn(l, pr.penalty) : __fdiv_rn(l, pr.penalty);
      if (before(l, v, pv, pi)) { pv = l; pi = v; }
    }
    kv[v] = l;
    ki[v] = v;
  }
  if (raw && gen < pr.logits_ld && gen == 0 && tid == 0) raw[((long)b * pr.logits_ld) * V + V - 1] = lg[(long)b * V + V - 1];
  block_argmax(pv, pi, shv, shi);
  const int pen_arg = pi;
  // block bitonic sort, descending
  for (int k = 2; k <= NS; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      __syncthreads();
      for (int i = tid; i < NS; i += blockDim.x) {
        const int o = i ^ j;
        if (o > i) {
          const bool desc = (i & k) == 0;
          const float a = kv[i], c = kv[o];
          const int ai = ki[i], ci = ki[o];
          if (desc ? before(c, ci, a, ai) : before(a, ai, c, ci)) { kv[i] = c; kv[o] = a; ki[i] = ci; ki[o] = ai; }
        }
      }
    }
  __syncthreads();
  // top-p: softmax of the sorted logits, inclusive cumsum, drop where cum > top_p (never the first)
  int K = Vv;
  if (pr.top_p < 1.f) {
    const float mx = kv[0];
    const int per = NS / blockDim.x > 0 ? NS / blockDim.x : 1;     // consecutive entries per thread
    float e[T2S_MAX_V / T2S_SAMPLE_THREADS];
    float loc = 0.f;
    for (int u = 0; u < per; ++u) {
      const int i = tid * per + u;
      e[u] = i < Vv ? expf(kv[i] - mx) : 0.f;
      loc += e[u];
    }
    const float tot = block_sum(loc, shv);
    float run = 0.f;
    for (int u = 0; u < per; ++u) { e[u] = e[u] / tot; run += e[u]; }
    // exclusive prefix of the per-thread sums
    const int lane = tid & 31, warp = tid >> 5;
    float incl = run;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    __syncthreads();
    if (lane == 31) scan[warp] = incl;
    __syncthreads();
    float wofs = 0.f;
    for (int w = 0; w < warp; ++w) wofs += scan[w];
    float cum = wofs + incl - run;
    int first_cut = 0x7fffffff;
    for (int u = 0; u < per; ++u) {
      const int i = tid * per + u;
      cum += e[u];
      if (i > 0 && i < Vv && cum > pr.top_p && i < first_cut) first_cut = i;
    }
    float fv = 0.f;
    int fi = first_cut;
    fv = -(float)first_cut;                       // argmax of -index = the smallest cut
    block_argmax(fv, fi, shv, shi);
    if (fi < K) K = fi;
  }
  const float temp = fmaxf(pr.temperature, 1e-5f);
  const int kk = min(pr.top_k, Vv);
  const float pivot = kk - 1 < K ? __fdiv_rn(kv[kk - 1], temp) : -INFINITY;
  __syncthreads();                                 // every warp has read kv[kk - 1] before the loop below overwrites it
  // final logits in sorted order, softmax, then argmax(probs / q) (first index on ties)
  float mx = -INFINITY;
  for (int i = tid; i < NS; i += blockDim.x) {
    float f = i < K ? __fdiv_rn(kv[i], temp) : -INFINITY;
    if (f < pivot) f = -INFINITY;
    kv[i] = f;
    mx = fmaxf(mx, f);
  }
  mx = warp_max(mx);
  __syncthreads();
  if ((tid & 31) == 0) scan[tid >> 5] = mx;
  __syncthreads();
  mx = scan[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmaxf(mx, scan[w]);
  float loc = 0.f;
  for (int i = tid; i < NS; i += blockDim.x) {
    const float e = kv[i] == -INFINITY ? 0.f : expf(kv[i] - mx);
    kv[i] = e;
    loc += e;
  }
  const float tot = block_sum(loc, shv);
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = tid; i < NS; i += blockDim.x) {
    if (i >= Vv) continue;
    const int v = ki[i];
    const float qv = q ? q[((long)b * pr.q_ld + gen) * V + v] : philox_exp(seeds[b], (uint32_t)gen, (uint32_t)v);
    const float sc = (kv[i] / tot) / qv;
    if (before(sc, v, bv, bi)) { bv = sc; bi = v; }
  }
  block_argmax(bv, bi, shv, shi);
  if (tid != 0) return;
  const int tok = bi, g = gen + 1;
  y[yoff + P + gen] = tok;
  seen[(long)b * ((V + 31) / 32) + (tok >> 5)] |= 1u << (tok & 31);
  s[ST_GEN] = g;
  const bool stop = (pr.early_stop != -1 && g > pr.early_stop) || pen_arg == V - 1 || tok == V - 1 || g >= pr.step_cap;
  if (stop) {
    s[ST_STOP] = 1;
    atomicAdd(n_stopped, 1);
  }
}

}  // namespace vtts
