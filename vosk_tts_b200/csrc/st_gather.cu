// st_gather.cu -- the gather of each token's BERT row into the StableTTS text phase (vtts_stabletts_synthesise_pieces_wav,
// engine.cu stt_bert_enqueue), declared in stabletts.cuh.
//
// A translation unit of its own so that engine.cu's module, which ptxas compiles as a whole, holds exactly the kernels it
// held before: every existing kernel keeps its machine code bit for bit (cuobjdump -sass).  The kernel does not stamp
// vtts_timeline (g_timeline lives in engine.cu's module).
#include <cuda_runtime.h>

namespace vtts {

// A copy, so the text phase reads exactly the rows a host gather of the same features would upload.  Waits for its
// predecessor, then lets its successor launch (the PDL order of kernels.cuh's PDL_WAIT).
__global__ void __launch_bounds__(128)
st_bert_gather_kernel(const float* __restrict__ feat, const int* __restrict__ src, int BD, float* __restrict__ bert,
                      const int* __restrict__ lens, const int* __restrict__ offs) {
  asm volatile("griddepcontrol.wait;\n\tgriddepcontrol.launch_dependents;" ::: "memory");
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= lens[b]) return;
  const long r = (long)offs[b] + t, s = src[r];
  for (int c = threadIdx.x; c < BD; c += blockDim.x) bert[r * BD + c] = feat[s * BD + c];
}

}  // namespace vtts
