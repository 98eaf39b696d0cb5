// st_tc.cu -- the plane-writing kernels of the StableTTS mel phase on the tensor cores (precision mode 2, engine.cu
// st_block_tc / st_enqueue), declared in dit.cuh.  Each is the dit.cuh kernel of the same name without "_planes", with the
// same fp32 arithmetic and the same fp32 outputs, and in addition writes the split-bf16 planes (hi, lo) of the rows that a
// tensor-core conv or attn_tc_kernel reads next.
//
// A translation unit of its own (like st_gather.cu) so that engine.cu's module, which ptxas compiles as a whole, holds
// exactly the kernels it held before: every existing kernel keeps its machine code bit for bit.  It therefore includes none
// of the engine's headers; the two helpers below restate theirs.  The kernels do not stamp vtts_timeline.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vtts {

namespace {

constexpr int LN_WARPS = 8;     // dit.cuh DIT_LN_WARPS: rows per CTA of the LayerNorm kernel (engine.cu launches 32 * 8 threads)
constexpr int LN_MAXV = 16;     // dit.cuh DIT_LN_MAXV: values per lane, hidden <= 512 (bind_stabletts refuses wider)

// Waits for the predecessor grid, then lets the successor launch (kernels.cuh PDL_WAIT).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;\n\tgriddepcontrol.launch_dependents;" ::: "memory"); }

// kernels.cuh split_bf16: hi = x rounded to bf16 on the bit pattern (ties away from zero), lo = the exact rest rounded the
// same way; the operand format every tensor-core conv of the engine reads.
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  const uint32_t h = (__float_as_uint(x) + 0x8000u) & 0xFFFF0000u;
  const float r = x - __uint_as_float(h);
  const uint32_t l = __float_as_uint(r) + 0x8000u;
  hi = __ushort_as_bfloat16((unsigned short)(h >> 16));
  lo = __ushort_as_bfloat16((unsigned short)(l >> 16));
}

__device__ __forceinline__ float silu(float v) { return v / (1.f + expf(-v)); }     // dit.cuh silu

}  // namespace

// dit_norm_kernel, plus the planes of `no` (pitch C): the operand of qkv and ffn1.
__global__ void __launch_bounds__(32 * LN_WARPS)
dit_norm_planes_kernel(const float* __restrict__ a, int lda, const float* __restrict__ film, const float* __restrict__ y, const float* __restrict__ ada,
                       int ada_ld, int gate_off, int shift_off, int scale_off, float eps, float* __restrict__ xo, float* __restrict__ no,
                       __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo, const int* __restrict__ lens,
                       const int* __restrict__ offs, int C) {
  pdl_wait();
  const int s = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * LN_WARPS + warp;
  if (t >= lens[s]) return;
  const long r = (long)offs[s] + t;
  const float* ad = ada + (long)s * ada_ld;
  float v[LN_MAXV];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
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
  for (int i = 0; i < LN_MAXV; ++i) {
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
  for (int i = 0; i < LN_MAXV; ++i) {
    const int c = lane + 32 * i;
    if (c < C) {
      const float o = __fadd_rn(__fmul_rn((v[i] - mean) * rstd, 1.f + ad[scale_off + c]), ad[shift_off + c]);
      no[r * C + c] = o;
      split_bf16(o, p_hi[r * C + c], p_lo[r * C + c]);
    }
  }
}

// dit_rope_kernel, plus the planes of the rotated q and k features (pitch 3 * heads * dk, the qkv planes attn_tc_kernel
// reads).  The planes of the features that pass through and of v are the qkv conv's epilogue output, left as they are.
__global__ void __launch_bounds__(128)
dit_rope_planes_kernel(float* __restrict__ qkv, const float2* __restrict__ tab, int heads, int dk, int d, __nv_bfloat16* __restrict__ p_hi,
                       __nv_bfloat16* __restrict__ p_lo, const int* __restrict__ lens, const int* __restrict__ offs) {
  pdl_wait();
  const int s = blockIdx.y, t = blockIdx.x;
  if (t >= lens[s]) return;
  const int hd = d / 2, HT = heads * dk;
  const long r0 = ((long)offs[s] + t) * 3 * HT;
  for (int i = threadIdx.x; i < 2 * heads * hd; i += blockDim.x) {
    const int j = i % hd, hq = i / hd;          // hq: head of q, then head of k
    const long p = r0 + (hq / heads) * HT + (hq % heads) * dk;
    const float2 cs = tab[(long)t * hd + j];
    const float a = qkv[p + j], b = qkv[p + j + hd];
    const float u = __fadd_rn(__fmul_rn(a, cs.x), __fmul_rn(-b, cs.y));
    const float w = __fadd_rn(__fmul_rn(b, cs.x), __fmul_rn(a, cs.y));
    qkv[p + j] = u;
    qkv[p + j + hd] = w;
    split_bf16(u, p_hi[p + j], p_lo[p + j]);
    split_bf16(w, p_hi[p + j + hd], p_lo[p + j + hd]);
  }
}

// dit_silu_kernel (in place), plus the planes of the result (pitch C): the operand of ffn2 and of cond_proj's second and
// third convs.
__global__ void __launch_bounds__(256)
dit_silu_planes_kernel(float* __restrict__ y, int C, __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo, const int* __restrict__ lens,
                       const int* __restrict__ offs) {
  pdl_wait();
  const int s = blockIdx.y, t = blockIdx.x;
  if (t >= lens[s]) return;
  const long r = ((long)offs[s] + t) * C;
  for (int c = threadIdx.x; c < C; c += 256) {
    const float v = silu(y[r + c]);
    y[r + c] = v;
    split_bf16(v, p_hi[r + c], p_lo[r + c]);
  }
}

// dit_gate_kernel, plus the planes of `out` at the same pitch ldo (p_hi / p_lo point at the same column block of the
// long-skip operand's planes as out does of its fp32 rows): the operand of the long-skip convs.
__global__ void __launch_bounds__(128)
dit_gate_planes_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ ada, int ada_ld, int gate_off,
                       float* __restrict__ out, int ldo, __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo,
                       const int* __restrict__ lens, const int* __restrict__ offs, int C) {
  pdl_wait();
  const int s = blockIdx.y, t = blockIdx.x;
  if (t >= lens[s]) return;
  const long r = (long)offs[s] + t;
  const float* g = ada + (long)s * ada_ld + gate_off;
  for (int c = threadIdx.x; c < C; c += 128) {
    const float v = __fadd_rn(x[r * C + c], __fmul_rn(g[c], y[r * C + c]));
    out[r * ldo + c] = v;
    split_bf16(v, p_hi[r * ldo + c], p_lo[r * ldo + c]);
  }
}

}  // namespace vtts
