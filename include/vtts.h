/*
 * vtts.h -- C ABI of the H100-native VITS2 inference engine (libvtts.so).
 *
 * Drop-in boundary: the single call the reference makes into its inference runtime,
 *
 *     audio = self.model.onnx.run(None, args)[0]        (vosk_tts/synth.py:123-126)
 *
 * on the session created at vosk_tts/model.py:46.  The graph behind that call is a trace of
 * SynthesizerTrn.infer (training/vits2/models.py:1679-1704, exported by
 * training/vits2/onnx_export.py:47-104) with feeds
 *     input int64[B,T], input_lengths int64[B], scales float32[3], sid int64[B]
 * and output float32[B,1,1,T_wav].  Every entry point below takes plain pointers and sizes
 * (no torch / numpy types); the Python facade in vosk_tts_b200/session.py binds them with
 * ctypes and exposes `run(None, feeds)`.
 *
 * All functions return VTTS_OK (0) or a negative status; the message of the last failure on a
 * handle is available through vtts_last_error().  Nothing throws across the ABI.  Calls on one
 * handle are serialised internally (InferenceSession.run is called concurrently by
 * server/tts_server.py:35,57), different handles are independent.
 */
#ifndef VTTS_H_
#define VTTS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VTTS_OK 0
#define VTTS_ERR_INVALID (-1)   /* bad argument / unsupported configuration           */
#define VTTS_ERR_CUDA (-2)      /* CUDA runtime failure (see vtts_last_error)          */
#define VTTS_ERR_WEIGHTS (-3)   /* tensor missing from / mis-sized in the weight blob   */
#define VTTS_ERR_CAPACITY (-4)  /* output buffer too small for the predicted durations   */
#define VTTS_ERR_STATE (-5)     /* vtts_synthesize without a preceding vtts_durations    */

typedef struct vtts_engine* vtts_handle;

/* Model hyper-parameters = the "model" block of the reference training json
 * (training/vits2/configs/mb_istft_vits2_multi.json:42-79) + the constants hard-coded in
 * SynthesizerTrn.__init__ (training/vits2/models.py:1613-1625). */
typedef struct vtts_config {
  int32_t n_vocab, n_speakers, gin_channels;
  int32_t inter_channels, hidden_channels, filter_channels;
  int32_t n_heads, n_layers, kernel_size, window_size;
  int32_t spk_cond_encoder, cond_layer_idx;
  int32_t use_transformer_flows;
  int32_t flow_kernel_size, flow_dilation_rate, flow_wn_layers, flow_n_flows;
  int32_t dp_filter_channels, dp_kernel_size, dp_n_flows, dp_num_bins;
  float dp_tail_bound;
  int32_t decoder_type;            /* 0 = Multiband_iSTFT_Generator, 1 = HiFi-GAN Generator */
  int32_t resblock_type;           /* 1 = ResBlock1, 2 = ResBlock2 */
  int32_t n_resblock_kernels;
  int32_t resblock_kernel_sizes[8];
  int32_t n_resblock_dilations;    /* dilations per resblock (same count for all) */
  int32_t resblock_dilations[8][8];
  int32_t n_upsamples;
  int32_t upsample_rates[8];
  int32_t upsample_kernel_sizes[8];
  int32_t upsample_initial_channel;
  int32_t subbands, istft_n_fft, istft_hop;
  int32_t precision;               /* 0 = fp32 FFMA everywhere; 1 = split-bf16 wgmma for the flow + decoder (dense convs and
                                      attention); 2 = text encoder on wgmma as well */
  int32_t flow_n_heads;            /* heads of the flow's pre_transformer: the reference hard-codes 2 (models.py:355) */
  /* Voice conversion (vtts_convert): input features of the posterior encoder enc_q (models.py:1616, mel_processing.py).
   * Only read when the blob carries enc_q (weights.pack(..., posterior=True)). */
  int32_t spec_channels;           /* enc_q input channels: n_mel_channels (mel) or filter_length/2+1 (linear spectrogram) */
  int32_t use_mel_posterior_encoder;
  int32_t filter_length, hop_length, win_length, n_mel_channels;
  float mel_fmin, mel_fmax;        /* (the mel filter bank itself is packed into the blob) */
  /* Model family of the blob: 0 = VITS2 SynthesizerTrn (every entry point above and below except the QuickVC ones),
   * 1 = QuickVC (vc/models.py; weights.pack_quickvc), which serves vtts_speaker_embedding* and vtts_quickvc_convert.  The entry points of one family
   * return VTTS_ERR_INVALID on an engine of the other. */
  int32_t model_family;
  /* ContentVec (HubertModel of vc/contentvec.py, transformers' HubertConfig; QuickVC engines whose blob carries cv.*):
   * vtts_content_units / vtts_quickvc_convert_wav.  cv_layers == 0: no ContentVec. */
  int32_t cv_layers, cv_hidden, cv_heads, cv_ffn;          /* transformer: 12 post-LN layers, 768 wide, 12 heads, FFN 3072 */
  int32_t cv_conv_dim, cv_n_conv;                          /* feature encoder: 7 convs of 512 channels */
  int32_t cv_conv_kernel[8], cv_conv_stride[8];            /* (10,3,3,3,3,2,2) / (5,2,2,2,2,2,2) */
  int32_t cv_pos_k, cv_pos_groups;                         /* positional conv: 128 taps, 16 groups */
  float cv_ln_eps, cv_gn_eps;                              /* LayerNorm eps (layer_norm_eps), layer 0's GroupNorm eps */
} vtts_config;

#define VTTS_FAMILY_VITS2 0
#define VTTS_FAMILY_QUICKVC 1

/* Replaces onnxruntime.InferenceSession(model.onnx) (vosk_tts/model.py:46).
 * `blob` holds the packed fp32 tensors produced by vosk_tts_b200.weights.pack(); `manifest` is a
 * NUL-terminated text table "name offset_in_floats numel\n".  `blob_is_device` != 0 means `blob`
 * is already a device pointer on `device` (e.g. the destination of an NCCL broadcast); the engine
 * then copies device-to-device.  The engine keeps its own copy either way. */
int vtts_create(const vtts_config* cfg, const float* blob, size_t blob_floats, const char* manifest,
                int blob_is_device, int device, vtts_handle* out);
void vtts_destroy(vtts_handle h);
const char* vtts_last_error(vtts_handle h);

/* Phase 1 of InferenceSession.run (models.py:1680-1691): speaker lookup, text encoder,
 * stochastic duration predictor, ceil'd durations.
 *   ids        int64 [B, t_max]   phoneme ids ("input"), rows padded arbitrarily beyond lengths
 *   lengths    int64 [B]          ("input_lengths")
 *   sid        int64 [B]          ("sid")
 *   scales     float [3]          noise_scale, length_scale, noise_scale_w ("scales")
 *   noise_dp   float [B,2,t_max]  replaces torch.randn at models.py:96, or NULL -> Philox(seed)
 *   y_lengths  out int64 [B]      frames per utterance (models.py:1691)
 *   durations  out int32 [B,t_max] w_ceil per token, or NULL
 * Host pointers.  Blocks until the lengths are known (the one data-dependent shape of the path). */
int vtts_durations(vtts_handle h, const int64_t* ids, const int64_t* lengths, const int64_t* sid,
                   int B, int t_max, const float* scales, const float* noise_dp, uint64_t seed,
                   int64_t* y_lengths, int32_t* durations);

/* Phase 2 (models.py:1692-1703): hard alignment, prior expansion + sampling, flow^-1, decoder.
 *   noise_z    float [B, inter_channels, z_ld]  replaces torch.randn_like at models.py:1700 (only the
 *              first y_lengths[b] columns of utterance b are read), or NULL -> Philox(seed)
 *   wav        out float [B, wav_ld]   utterance b occupies wav[b*wav_ld .. + hop*y_lengths[b])
 *   frame_token out int32 [B, idx_ld]  frame -> token index (the alignment `attn`, models.py:1694), or NULL
 * Host pointers.  Returns VTTS_ERR_CAPACITY if wav_ld < hop*max(y_lengths). */
int vtts_synthesize(vtts_handle h, const float* noise_z, int z_ld, float* wav, int64_t wav_ld,
                    int32_t* frame_token, int idx_ld);

/* Same two phases with device-resident inputs/outputs (pointers on the engine's device):
 * used to time the path without host<->device copies.  The layouts match the host variants. */
int vtts_durations_dev(vtts_handle h, const int64_t* d_ids, const int64_t* lengths_host, const int64_t* d_sid,
                       int B, int t_max, const float* scales, const float* d_noise_dp, uint64_t seed,
                       int64_t* y_lengths_host);
int vtts_synthesize_dev(vtts_handle h, const float* d_noise_z, int z_ld, float* d_wav, int64_t wav_ld);

/* Both phases in one call (== one InferenceSession.run).  The caller provides capacity instead of exact sizes:
 * z_ld columns of noise_z (if given) and wav_ld samples per utterance; VTTS_ERR_CAPACITY is returned after phase 1
 * (y_lengths filled in, durations kept) when they are too small, and vtts_synthesize can then be called with
 * larger buffers. */
int vtts_infer(vtts_handle h, const int64_t* ids, const int64_t* lengths, const int64_t* sid, int B, int t_max,
               const float* scales, const float* noise_dp, const float* noise_z, int z_ld, uint64_t seed,
               int64_t* y_lengths, float* wav, int64_t wav_ld, int32_t* frame_token, int idx_ld);
int vtts_infer_dev(vtts_handle h, const int64_t* d_ids, const int64_t* lengths_host, const int64_t* d_sid, int B, int t_max,
                   const float* scales, const float* d_noise_dp, const float* d_noise_z, int z_ld, uint64_t seed,
                   int64_t* y_lengths_host, float* d_wav, int64_t wav_ld);

/* Streaming synthesis of one long utterance (BASELINE.json configs[4]): after vtts_durations, vtts_flow runs the
 * alignment, sampling and the flow once; vtts_decode_chunk then vocodes latent frames [f0, f1) with a
 * vtts_decoder_halo()-frame halo on each side that is computed and discarded ("overlap-discard": exact, because the
 * halo covers the decoder's receptive field), so audio can be handed out chunk by chunk.  B must be 1.
 * wav receives hop*(f1-f0) samples. */
int vtts_decoder_halo(vtts_handle h);
int vtts_flow(vtts_handle h, const float* noise_z, int z_ld);
int vtts_decode_chunk(vtts_handle h, int f0, int f1, float* wav, int64_t wav_capacity);

/* Samples produced per latent frame (256 for the reference config). */
int vtts_hop(vtts_handle h);
/* CUDA-event time (ms) of each stage of the last call: [0] encoder, [1] duration predictor +
 * regulator, [2] prior sampling + flow, [3] decoder, [4] H2D, [5] D2H.  n <= 8. */
int vtts_stage_timings(vtts_handle h, float* ms, int n);
/* Number of kernels this engine launched since creation (bench.py's gpu_launches). */
uint64_t vtts_kernel_launches(vtts_handle h);
/* The CUDA stream (cudaStream_t as void*) the engine launches on, for external event timing. */
void* vtts_stream(vtts_handle h);
/* Runs one named kernel micro-benchmark on the engine's device; see csrc/engine.cu. Returns ms or <0. */
float vtts_microbench(vtts_handle h, const char* what, int iters);

/* CUDA graphs (default on): a call shape (batch, lengths) seen before is captured once and replayed, which removes
 * the ~160 per-call kernel-launch overheads at batch 1.  vtts_graph_replays counts graph launches so far. */
int vtts_set_graphs(vtts_handle h, int enable);
uint64_t vtts_graph_replays(vtts_handle h);
/* Single-utterance vtts_infer / vtts_infer_dev calls enqueue the second phase for a PREDICTED length bucket without waiting
 * for the durations (the kernels read the true lengths on the device) and repeat it only when the prediction was too small:
 * hits / misses since creation. */
int vtts_speculation_stats(vtts_handle h, uint64_t* hits, uint64_t* misses);
/* Host-side wall clock (microseconds) of the last single-utterance vtts_infer call: [0] phase-1 enqueue, [1] phase-2 +
 * copy-back enqueue, [2] wait for the stream, [3] copy-out, [4] total, [5] 1 = speculative hit, 2 = miss, 0 = not speculative. */
int vtts_host_timings(vtts_handle h, double* us, int n);

/* Per-launch profiling of the dense-conv kernel family (the dominant kernels): while enabled every launch is
 * bracketed by CUDA events on the engine's stream.  vtts_profile_read returns the summed device time, the
 * number of launches and the algorithmic FLOPs (2*Cin*k*Cout per output position) since vtts_profile(h,1). */
int vtts_profile(vtts_handle h, int enable);
int vtts_profile_read(vtts_handle h, double* conv_ms, uint64_t* conv_launches, double* conv_flops);
/* Same counters for the tensor-core conv kernel (precision mode 1). */
int vtts_profile_read_tc(vtts_handle h, double* ms, uint64_t* launches, double* flops);

/* In-graph timeline for tuning: enable=1 arms it, enable=0 disarms, enable=2 reads up to max_pairs (source line,
 * %globaltimer ns) pairs -- one per kernel launch, stamped by the kernel's first CTA at entry. */
int vtts_timeline(vtts_handle h, int enable, unsigned long long* out, size_t max_pairs, size_t* n_out);

/* Test hooks: flags bit0 keeps a copy of z_p (models.py:1700); vtts_debug_read copies a named workspace
 * tensor of the last call ("x", "stats", "dx", "za", "zb", "condv", "z_p", "z", "d0", "stage<i>", "post") to
 * host memory in the engine's channels-last packed layout.  After a conversion: "vc_spec" (enc_q input rows: the log-mel or
 * linear spectrogram, spec_channels rounded up to 16 columns), "vc_z" (posterior sample) and "vc_z_p" (flow forward output;
 * both kept when bit0 is set), "vc_z_hat" (flow reverse output).  After a speaker embedding (QuickVC): "vc_spec" (log-mel
 * rows), "spk_x<l>" (projected LSTM inputs of layer l, [rows][1024]: frame rows for l = 0, slice rows for l = 1, 2),
 * "spk_h<l>" (hidden states of layer l, slice rows [rows][256]: the slices in clip order, each occupying as many rows as it
 * has frames, 8 rows between consecutive slices) and "spk_g". */
int vtts_debug_flags(vtts_handle h, int flags);
int vtts_debug_read(vtts_handle h, const char* name, float* out, size_t max_floats, size_t* n_out);
/* Unit-test hook for the relative-position attention kernels (attentions.py:165-196): ONE attention launch of layer
 * "enc.<i>" or "flow.<f>.tr" through the engine's own launch code, on host tensors.
 *   B, lens          utterances, packed as the engine packs them: utterance b starts at row offs[b], SEQ_GAP (8) rows between
 *                    consecutive utterances
 *   launch_lens      per-utterance lengths >= lens the launch is sized for (the bucket lengths of a captured graph: grid,
 *                    maxLen and the kernel heuristics see them, the kernels read lens), or NULL = lens
 *   qkv              fp32 [rows][3H], every row: gap rows and rows behind the last utterance hold whatever the caller put there.
 *                    The tensor-core kernel reads the split-bf16 planes of all rows, taken from the engine's plane pool and
 *                    cleared behind each utterance by the production zero_tails pass, as a phase does
 *   kernel           VTTS_ATTN_AUTO (the engine's choice), _TC (attn_tc_kernel), _SPLIT (attn_split_kernel), _R1 / _R4
 *                    (attn_kernel with 1 / 4 query rows per warp), _FFMA (the engine's choice among the FFMA kernels)
 *   out              fp32 [rows][H] (in/out: rows outside the utterances are left as they are), or NULL
 *   planes           uint16 [p_planes][rows * H] (in/out) split-bf16 planes of the output (hi, lo) or (hi, mid, lo), or NULL;
 *                    the tensor-core kernel writes 2 planes only.  At least one of out / planes.
 *   iters > 0        *ms_out = average device time of `iters` more launches
 *   report           out: the launch that ran
 * A kernel the layer cannot run (tensor cores without the split-bf16 relative tables or with 2W+1 > 13, split-KV where the
 * key tiles do not fit shared memory or the CTAs one wave) and malformed arguments return VTTS_ERR_INVALID before any launch.
 * The engine's kernel selection settings are restored on every exit. */
#define VTTS_ATTN_AUTO 0
#define VTTS_ATTN_TC 1
#define VTTS_ATTN_SPLIT 2
#define VTTS_ATTN_R1 3
#define VTTS_ATTN_R4 4
#define VTTS_ATTN_FFMA 5
typedef struct vtts_attn_report {
  int kernel;                   /* VTTS_ATTN_TC / _SPLIT / _R1 / _R4 */
  int dk;                       /* head width: the kernel's template */
  int R;                        /* query rows per warp (FFMA kernels) */
  int grid_x, grid_y, grid_z;
  int smem;                     /* dynamic shared memory bytes */
} vtts_attn_report;
int vtts_debug_attention(vtts_handle h, const char* layer, int B, const int* lens, const int* launch_lens, const float* qkv,
                         size_t rows, int kernel, float* out, uint16_t* planes, int p_planes, int iters, float* ms_out,
                         vtts_attn_report* report);

/* Unit-test hook for the dense conv kernels: ONE grouped launch of the tensor-core conv (conv_tc.cuh) or of the fp32 FFMA
 * conv (kernels.cuh conv_kernel) through the engine's own launch code, on host tensors.
 *   B, lens, rmul    utterance b has lens[b] * rmul input rows; utterances are packed as the engine packs them
 *                    (SEQ_GAP = 8 rows between utterances, scaled by rmul, plus in_extra / out_seq_extra per utterance)
 *   problems         1..4 problems of the launch (vtts_conv_problem)
 *   x, x_n           tensor cores: x_planes (2 or 3) bf16 planes [x_n rows][Cin] back to back (hi, lo or hi, mid, lo), shared
 *                    by every problem; copied into the engine's plane pool, whose rows behind each utterance are then
 *                    zeroed as at the start of a phase.  FFMA: x_n fp32 values, problem-specific ldx / xoff.
 *   y, y_n           in/out fp32 buffer every problem with y_on writes to (its prior contents are uploaded, so rows a
 *                    kernel must not touch keep what the caller wrote, and res == 2 reads it as the residual)
 *   res, res_n       fp32 residual buffer of the problems with res == 1
 *   p_out, p_n       in/out split-bf16 output planes, p_planes (2 or 3) planes of p_n elements back to back (hi, lo or
 *                    hi, mid, lo), written by the problems with planes_on as split(lrelu(out, pl_slope))
 *   ov               launch-shape overrides for this call only (VTTS_CONV_KEEP: the engine's setting), or NULL
 *   report           out: the launch that ran
 * Malformed specs (channel counts the kernel cannot take, more than 4 problems, mixed plane counts, halos the packed layout
 * or the FFMA tile cannot hold, buffers too small for the rows a problem writes or reads) return VTTS_ERR_INVALID before
 * anything is launched.  Tensor cores need a precision >= 1 engine. */
#define VTTS_CONV_KEEP (-1000000)
typedef struct vtts_conv_problem {
  int Cin, Cout, k, dil, pad;
  int out_mul, out_add;         /* output row of input position t: t * out_mul + out_add (polyphase ConvTranspose1d) */
  int in_extra, out_seq_extra;  /* extra logical input rows / extra output rows per utterance */
  int epi;                      /* 1 ReLU, 2 gate (tanh(even) * sigmoid(odd) channel pairs), 4 tanh (FFMA only) */
  float alpha, pl_slope;        /* out = act(conv + bias + cond) * alpha + res; planes of lrelu(out, pl_slope) */
  const uint16_t *w_hi, *w_mid, *w_lo;  /* tensor cores: bf16 [k][Cout][Cin] (w_mid for 3-plane launches only) */
  const float* w;               /* FFMA: [k][Cin][ldw], ldw = (Cout + 3) / 4 * 4 */
  const float* bias;            /* [Cout] (FFMA: [ldw]) */
  const float* cond;            /* optional [B][cond_ld], added to the bias of utterance b */
  int cond_ld;
  int y_on, ldy, yoff;
  int res, ldr, roff;           /* 0 none, 1 the res buffer, 2 the y buffer itself (in place) */
  int planes_on, ldp, poff;     /* poff: tensor cores only */
  int ldx, xoff, reflect, pro;  /* FFMA input: row pitch / column offset, ReflectionPad1d((1,0)) row map, 1 = leaky-ReLU prologue */
  float slope;
} vtts_conv_problem;
typedef struct vtts_conv_overrides {
  int tc_bn, tc_split, tc_tall, tc_mc, tc_persist, tc_wmc, tc_min_steps, conv_max_s, conv_min_g, conv_max_g, conv_big_g;
} vtts_conv_overrides;
typedef struct vtts_conv_report {
  int use_tc;
  int bn, split, tall, cn, wmc, persist, np, ast, wst;
  int image;                    /* 0 conv_tc_kernel<BN, false>, 1 conv_tc_kernel<BN, true>, 2 conv_tc_persist_kernel<BN> */
  int S, G;                     /* FFMA: cluster split-K and thread groups */
  int grid_x, grid_y, grid_z;
  int psplit[4];                /* tensor cores: split-K of each problem's tiles (dividing `split`, the cluster size; 0 past the
                                   last problem).  Problems with psplit < split share a cluster between split / psplit tiles,
                                   and the grid is then (1, 1, clusters * split) */
} vtts_conv_report;
int vtts_debug_conv(vtts_handle h, int use_tc, int B, const int* lens, int rmul, int n_problems, const vtts_conv_problem* problems,
                    const void* x, size_t x_n, int x_planes, float* y, size_t y_n, const float* res, size_t res_n, uint16_t* p_out,
                    size_t p_n, int p_planes, const vtts_conv_overrides* ov, vtts_conv_report* report);
/* Launch-shape log of the dense conv launches: mode 1 clears and starts it, 0 stops it, 2 copies up to max_n entries (one
 * per launch the host enqueued since it was started; graph replays enqueue none) and sets *n_out. */
int vtts_debug_conv_log(vtts_handle h, int mode, vtts_conv_report* out, int max_n, int* n_out);
/* The split-K plan the engine makes for one grouped tensor-core conv launch, computed on the host alone (no device, no
 * engine).  Problems p < n (1..4): cin[p] (a multiple of 64), cout[p], k[p], in_extra[p]; B utterances of lens[b] <= max_len
 * rows / rmul; bn 64 / 128 pins the tile width (0: either); max_split caps the cluster size (8: none); min_steps = k-steps
 * per split CTA at least; n_sm and cluster_cap (co-resident clusters of 2/4/8 CTAs at BN 64, then at BN 128) describe the
 * device.  plan (out, 6 ints): BN, cluster size, and the split of each problem (0 past the last). */
int vtts_tc_split_plan(int n, const int* cin, const int* cout, const int* k, const int* in_extra, int B, const int* lens,
                       int rmul, int max_len, int bn, int max_split, int min_steps, int n_sm, const int* cluster_cap, int* plan);

/* Voice conversion (SynthesizerTrn.voice_conversion, models.py:1710-1718): re-voices recordings of speaker sid_src as
 * speaker sid_tgt of the same multi-speaker model.  One call = spectrogram front end, posterior encoder enc_q (g_src),
 * flow forward (g_src), flow reverse (g_tgt), decoder (g_tgt); no host synchronisation inside (the frame counts follow
 * from the input lengths: frames = (len + 2*pad - filter_length) / hop_length + 1, pad = (filter_length - hop_length) / 2,
 * i.e. len / 256 for the reference configuration).
 *   wav          float [B, wav_ld] in [-1, 1], clip b = wav[b*wav_ld .. + wav_lengths[b]); every clip is padded and framed
 *                on its own samples; needs wav_lengths[b] > pad (385 samples for the reference configuration)
 *   noise_scale  scales the posterior's eps (the reference uses 1); 0 gives z = m
 *   noise_q      float [B, inter_channels, q_ld] replaces torch.randn_like at models.py:841 (columns < frames[b] read), or
 *                NULL -> Philox(seed)
 *   out_wav      out float [B, out_ld]: clip b gets hop * out_frames[b] samples
 *   out_frames   out int64 [B]
 * Host pointers, atomic on the handle.  VTTS_ERR_INVALID: the blob has no enc_q, n_speakers <= 1, a speaker id out of range,
 * a clip too short for the reflect padding, or an odd flow_n_flows (the Flip folding of the packed flow is only valid for
 * both directions with an even count).  VTTS_ERR_CAPACITY: out_ld < hop * max(frames). */
int vtts_convert(vtts_handle h, const float* wav, const int64_t* wav_lengths, int B, int64_t wav_ld, const int64_t* sid_src,
                 const int64_t* sid_tgt, float noise_scale, const float* noise_q, int q_ld, uint64_t seed, float* out_wav,
                 int64_t out_ld, int64_t* out_frames);
/* Same without the front end: spec float [B, spec_channels, spec_ld] is the reference's `y` (log-mel or linear magnitude
 * spectrogram), spec_lengths[b] frames valid (1 <= spec_lengths[b] <= spec_ld). */
int vtts_convert_spec(vtts_handle h, const float* spec, const int64_t* spec_lengths, int B, int64_t spec_ld, const int64_t* sid_src,
                      const int64_t* sid_tgt, float noise_scale, const float* noise_q, int q_ld, uint64_t seed, float* out_wav,
                      int64_t out_ld, int64_t* out_frames);

/* Forced alignment: the text-to-frame alignment at the head of SynthesizerTrn.forward (models.py:1632-1660).  One call =
 * text encoder enc_p on the ids (speaker sid), spectrogram front end, enc_q and the forward flow on the recording (g = the
 * same speaker; none for a single-speaker model, n_speakers <= 1, where sid may be NULL), the Gaussian log-likelihood
 * neg_cent of every frame under every token's prior, and Monotonic Alignment Search; no host synchronisation inside.  The
 * noise-scaled MAS of models.py:1653-1655 (a training regulariser) is never added.
 *   ids          int64 [B, t_max], id_lengths[b] tokens valid (1 <= t_x <= min(t_max, 2048, frames[b]))
 *   wav ... seed as vtts_convert: noise_scale 1 is the reference's forward, 0 aligns the posterior mean
 *   durations    out int32 [B, t_max]: frames of each token (the reference's w = attn.sum(2)), 0 past id_lengths[b]
 *   token_of_frame  out int32 [B, tof_ld] or NULL: the token each frame is aligned to, -1 past out_frames[b]
 *   score        out float [B] or NULL: log-likelihood of the best path (sum of neg_cent along it, fp32)
 *   out_frames   out int64 [B]
 * Host pointers, atomic on the handle.  VTTS_ERR_INVALID: the blob has no enc_q (model.onnx never has it: pack with
 * posterior=True), an odd flow_n_flows, a phoneme id out of [0, n_vocab), a speaker id out of range for a multi-speaker
 * model, a clip too short for the reflect padding, t_x < 1, t_x > frames (no monotonic path exists) or t_x > 2048.
 * VTTS_ERR_CAPACITY: tof_ld < max(frames) or q_ld < max(frames). */
int vtts_align(vtts_handle h, const int64_t* ids, const int64_t* id_lengths, int t_max, const int64_t* sid, const float* wav,
               const int64_t* wav_lengths, int B, int64_t wav_ld, float noise_scale, const float* noise_q, int q_ld, uint64_t seed,
               int32_t* durations, int32_t* token_of_frame, int64_t tof_ld, float* score, int64_t* out_frames);
/* Same from the posterior encoder's input features: spec float [B, spec_channels, spec_ld], spec_lengths[b] frames valid. */
int vtts_align_spec(vtts_handle h, const int64_t* ids, const int64_t* id_lengths, int t_max, const int64_t* sid, const float* spec,
                    const int64_t* spec_lengths, int B, int64_t spec_ld, float noise_scale, const float* noise_q, int q_ld, uint64_t seed,
                    int32_t* durations, int32_t* token_of_frame, int64_t tof_ld, float* score, int64_t* out_frames);

/* QuickVC speaker embedding (SpeakerEncoder.embed_utterance, vc/models.py:728-767, as SynthesizerTrn.infer calls it on the
 * target's mel_spectrogram_torch): the g a conversion is conditioned on, from a recording of any speaker.  A clip of T <= 128
 * mel frames is one sequence of T frames; a longer one is cut into 128-frame slices starting at 0, 64, ... < T - 128, plus
 * its last 128 frames; the 3-layer LSTM runs over every slice, each slice's final hidden state goes through linear, ReLU
 * and L2 normalisation, and g is the mean over the clip's slices.  One call, no host synchronisation inside.
 *   wav          float [B, wav_ld] in [-1, 1] at the model's sampling rate (16 kHz), clip b = wav[b*wav_ld .. +
 *                wav_lengths[b]); each clip is framed on its own samples (frames = (len + 2*pad - filter_length) / hop_length
 *                + 1, pad = (filter_length - hop_length) / 2), and needs wav_lengths[b] > pad (480 samples at the published
 *                configuration)
 *   g_out        out float [B, gin_channels]
 * Host pointers, atomic on the handle.  VTTS_ERR_INVALID: not a QuickVC engine, a clip too short for the reflect padding. */
int vtts_speaker_embedding(vtts_handle h, const float* wav, const int64_t* wav_lengths, int B, int64_t wav_ld, float* g_out);
/* Same from log-mel rows: mel float [B, n_mel_channels, mel_ld] (the reference's mel_spectrogram_torch output),
 * mel_lengths[b] frames valid (1 <= mel_lengths[b] <= mel_ld). */
int vtts_speaker_embedding_mel(vtts_handle h, const float* mel, const int64_t* mel_lengths, int B, int64_t mel_ld, float* g_out);

/* QuickVC conversion (SynthesizerTrn.infer, vc/models.py:862-872, as vc/convert.py:62-87 calls it) of content units into the
 * voice of a target: z_p = enc_p(units) (PosteriorEncoder(768, I, H, 5, 1, 16), no g), z = flow(z_p, g, reverse=True),
 * o = dec(z, g) (Multistream_iSTFT_Generator: x = conv_pre(z) + cond(g), the inverse STFT divided by the window envelope as
 * torch.istft does).  Each clip is converted as if alone.  One call, no host synchronisation inside.
 *   units        float [B, units_ld, 768], frame-major (ContentVec's last_hidden_state, vc/encode.py's [T, 768] .npy rows);
 *                clip b = its first unit_lengths[b] frames, 1 <= unit_lengths[b] <= units_ld
 *   g            float [B, gin_channels]: the target's speaker embedding (vtts_speaker_embedding; a target is enrolled once
 *                and reused across sources)
 *   noise_scale  scales enc_p's sample: 1 is the reference (z_p = m + eps * exp(logs)), 0 gives z_p = m
 *   noise        float [B, inter_channels, noise_ld] standing in for torch.randn_like (vc/models.py:270), or NULL for Philox(seed)
 *   out_wav      out float [B, out_ld]: clip b gets hop * unit_lengths[b] samples (320 per 20 ms unit at the published
 *                configuration), zeros after them;  out_frames out int64 [B] = unit_lengths
 * Host pointers, atomic on the handle.  Precision modes 2 and 3 run as mode 1 (they differ only in the VITS2 text encoder).
 * VTTS_ERR_INVALID: not a QuickVC engine, a blob without the conversion tensors (speaker encoder only), B < 1, a length outside
 * [1, units_ld], g NULL.  VTTS_ERR_CAPACITY: out_ld < hop * max(unit_lengths), noise_ld < max(unit_lengths).
 * After a call, vtts_debug_read "vc_z" (bit0 of vtts_debug_flags set) is z_p and "vc_z_hat" is z, frame rows [rows][inter]. */
int vtts_quickvc_convert(vtts_handle h, const float* units, const int64_t* unit_lengths, int B, int64_t units_ld,
                         const float* g, float noise_scale, const float* noise, int noise_ld, uint64_t seed,
                         float* out_wav, int64_t out_ld, int64_t* out_frames);

/* ContentVec content units (HubertModel(...)["last_hidden_state"], as vc/encode.py and vc/convert.py:82 compute them) of
 * 16 kHz source recordings.  Each clip is processed as if alone (B = 1 in the reference).  Frames per clip: L0 = (len - K0) / s0
 * + 1, then L_i = (L_{i-1} - k_i) / s_i + 1 (499 for 10 s; a clip needs at least 400 samples at the published shape).
 *   wav        float [B, wav_ld] in [-1, 1], clip b = its first wav_lengths[b] samples (no normalisation, as convert.py)
 *   units      out float [B, units_ld, cv_hidden], frame-major (vtts_quickvc_convert's input layout), zeros after each clip
 *   out_frames out int64 [B]
 * Host pointers, atomic on the handle; one graphed call keyed by batch and sample-length bucket.  Every stage runs on the fp32
 * FFMA pipe in every precision mode.  VTTS_ERR_INVALID: not a QuickVC engine, a blob without cv.*, B < 1, a clip too short
 * for one frame or longer than wav_ld.  VTTS_ERR_CAPACITY: units_ld below a clip's frame count.
 * After a call with bit0 of vtts_debug_flags set, vtts_debug_read "cv_feat" is the feature encoder's output [rows][cv_conv_dim]
 * and "cv_enc_in" the transformer's input (after the positional conv and its LayerNorm) [rows][cv_hidden]; clip 0 starts
 * at row 0. */
int vtts_content_units(vtts_handle h, const float* wav, const int64_t* wav_lengths, int B, int64_t wav_ld, float* units,
                       int64_t units_ld, int64_t* out_frames);
/* Source recordings -> waveforms in the voice of g: vtts_content_units, then vtts_quickvc_convert on its units, in ONE call
 * (the last LayerNorm writes the rows enc_p reads).  Arguments as those two; noise [B, inter_channels, noise_ld] with
 * noise_ld >= the largest frame count, out_ld >= hop * that count.  VTTS_ERR_INVALID also for a blob without the conversion
 * tensors. */
int vtts_quickvc_convert_wav(vtts_handle h, const float* wav, const int64_t* wav_lengths, int B, int64_t wav_ld, const float* g,
                             float noise_scale, const float* noise, int noise_ld, uint64_t seed, float* out_wav, int64_t out_ld,
                             int64_t* out_frames);

/* Monotonic Alignment Search on the GPU -- replaces monotonic_align.maximum_path (training/vits2/monotonic_align/__init__.py:6-22,
 * core.pyx:7-43; called from SynthesizerTrn.forward, models.py:1658).  Handle-free (no engine state); errors of these two are
 * read with vtts_last_error(NULL) on the calling thread.
 * neg_cent: float32 [B][T_y][T_x] scores (frames x tokens, as the reference passes them); t_ys / t_xs: valid frames / tokens
 * per item (the reference derives them from the mask sums), 0 <= t_x <= t_y required; path: int32 [B][T_y][T_x], 1 on the path.
 * Host pointers; runs on `device`.  The _dev variant takes device pointers, overwrites d_value with the accumulated scores
 * (like the reference's in-place update) and only enqueues on `stream` (a cudaStream_t, may be NULL). */
int vtts_maximum_path(const float* neg_cent, const int32_t* t_ys, const int32_t* t_xs, int B, int T_y, int T_x, int32_t* path,
                      int device);
int vtts_maximum_path_dev(float* d_value, const int32_t* d_t_ys, const int32_t* d_t_xs, int B, int T_y, int T_x, int32_t* d_path,
                          void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VTTS_H_ */
