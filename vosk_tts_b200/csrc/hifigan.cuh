// hifigan.cuh -- the hand-off from StableTTS's mel phase to its vocoder (the HiFi-GAN Generator, matcha/hifigan/models.py:
// 148-206, which runs on the decoder kernels of kernels.cuh and conv_tc.cuh).
#pragma once
#include "kernels.cuh"

namespace vtts {

// The vocoder's input rows: the first B (conditional) sequences of the mel phase, denormalised (mel * mel_std + mel_mean, in the
// reference's two fp32 roundings, matcha/utils/model.py) unless the phase already wrote them so (prm[2] != 0).  Rows past
// each utterance's frame count are not written: the vocoder's convs read zeros there.
__global__ void hg_mel_in_kernel(const float* __restrict__ mel, int NC, const float* __restrict__ prm, const float* __restrict__ mel_mean,
                                 const float* __restrict__ mel_std, float* __restrict__ out, const int* __restrict__ lens,
                                 const int* __restrict__ offs) {
  PDL_LAUNCH();
  PDL_WAIT();
  const int b = blockIdx.y, t = blockIdx.x;
  if (t >= lens[b]) return;
  const long r = (long)offs[b] + t;
  const bool den = prm[2] != 0.f;
  for (int c = threadIdx.x; c < NC; c += blockDim.x) {
    const float x = mel[r * NC + c];
    out[r * NC + c] = den ? x : __fadd_rn(__fmul_rn(x, mel_std[0]), mel_mean[0]);
  }
}

}  // namespace vtts
