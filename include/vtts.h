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
                                      attention); 2 = text encoder on wgmma as well.  StableTTS: 1 = vocoder and BERT on
                                      wgmma; 2 = also the flow-matching decoder's convs (where their widths are multiples
                                      of 64) and attention, from the split-bf16 weights weights.pack_stabletts*(...,
                                      precision=2) adds; its text phase stays fp32 FFMA in every mode */
  int32_t flow_n_heads;            /* heads of the flow's pre_transformer: the reference hard-codes 2 (models.py:355) */
  /* Voice conversion (vtts_convert): input features of the posterior encoder enc_q (models.py:1616, mel_processing.py).
   * Only read when the blob carries enc_q (weights.pack(..., posterior=True)). */
  int32_t spec_channels;           /* enc_q input channels: n_mel_channels (mel) or filter_length/2+1 (linear spectrogram) */
  int32_t use_mel_posterior_encoder;
  int32_t filter_length, hop_length, win_length, n_mel_channels;
  float mel_fmin, mel_fmax;        /* (the mel filter bank itself is packed into the blob) */
  /* Model family of the blob: 0 = VITS2 SynthesizerTrn (every entry point above and below except the QuickVC ones),
   * 1 = QuickVC (vc/models.py; weights.pack_quickvc), which serves vtts_speaker_embedding* and vtts_quickvc_convert,
   * 2 = StableTTS (weights.pack_stabletts_cfm: the flow-matching decoder, which serves vtts_cfm_decode; weights.pack_stabletts:
   * the text encoder as well, which also serves vtts_stabletts_synthesise).  The entry points of one family return
   * VTTS_ERR_INVALID on an engine of another.  3 = GPT-SoVITS text-to-semantic decoder (weights.pack_t2s), which serves
   * vtts_t2s_decode.  4 = GPT-SoVITS SoVITS (weights.pack_sovits: HuBERT, ssl_proj and the quantizer's codebook), which
   * serves vtts_sovits_semantic and vtts_sovits_latent. */
  int32_t model_family;
  /* StableTTS flow-matching decoder (model_family 2; CFM of training/stabletts/matcha/models/components/flow_matching.py:301,
   * weights.pack_stabletts_cfm): vtts_cfm_decode.  The other families leave these 0. */
  int32_t st_noise, st_cond, st_hidden, st_filter;         /* mel channels 80, encoder output 256, hidden 384, FFN / prenet 768 */
  int32_t st_layers, st_heads, st_kernel;                  /* 6 DitWrapper blocks (even: U-Net long skips), 4 heads, k = 3 */
  int32_t st_spk_dim, st_n_spks;                           /* speaker embedding width 128, rows of spk_emb */
  /* StableTTS text encoder and durations (TextEncoder of components/text_encoder.py:55-139; model_family 2 blobs of
   * weights.pack_stabletts): vtts_stabletts_synthesise.  st_enc_layers == 0: the blob holds the decoder only. */
  int32_t st_n_vocab, st_streams;                          /* rows of emb / punc_emb; id streams per token: 5 (1 + 4 punctuation) */
  int32_t st_emb_dim, st_punc_dim, st_bert_dim, st_bert_proj;  /* 160, 16, 768 -> 32: 160 + 4 x 16 + 32 = st_cond */
  int32_t st_enc_hidden, st_enc_filter, st_enc_layers, st_enc_heads, st_enc_kernel;  /* both stacks: 256, 1024, 4 blocks, 4 heads, k = 3 */
  int32_t st_dur_channels;                                 /* dp_encoder's proj: 50 channels whose sigmoids sum to a duration */
  /* ContentVec (HubertModel of vc/contentvec.py, transformers' HubertConfig; QuickVC engines whose blob carries cv.*):
   * vtts_content_units / vtts_quickvc_convert_wav.  cv_layers == 0: no ContentVec. */
  int32_t cv_layers, cv_hidden, cv_heads, cv_ffn;          /* transformer: 12 post-LN layers, 768 wide, 12 heads, FFN 3072 */
  int32_t cv_conv_dim, cv_n_conv;                          /* feature encoder: 7 convs of 512 channels */
  int32_t cv_conv_kernel[8], cv_conv_stride[8];            /* (10,3,3,3,3,2,2) / (5,2,2,2,2,2,2) */
  int32_t cv_pos_k, cv_pos_groups;                         /* positional conv: 128 taps, 16 groups */
  float cv_ln_eps, cv_gn_eps;                              /* LayerNorm eps (layer_norm_eps), layer 0's GroupNorm eps */
  /* In StableTTS engines whose blob carries bt.* (BERT: vtts_bert_features) the cv_* fields above describe BERT's transformer:
   * cv_layers the layers that run (the exported graph returns hidden_states[-3], so n_layers - 2 of a checkpoint), cv_hidden,
   * cv_heads, cv_ffn and cv_ln_eps (1e-12).  The rows of the word, position and token-type tables are those of the blob's
   * bt.emb.word / .pos / .type.
   * In GPT-SoVITS text-to-semantic engines (model_family 3) they describe the GPT's post-LN layers: cv_layers (n_layer),
   * cv_hidden (hidden_dim = embedding_dim), cv_heads (head), cv_ffn (4 hidden_dim) and cv_ln_eps (1e-5); the phone and semantic
   * vocabularies and the positions are the rows of the blob's t2s.temb / t2s.aemb / t2s.pe.
   * In GPT-SoVITS SoVITS engines (model_family 4) they describe chinese-hubert-base (a HubertModel of ContentVec's shape), and
   * n_vocab is the entry count of the quantizer's codebook (1024): the semantic tokens' vocabulary. */
} vtts_config;

#define VTTS_FAMILY_VITS2 0
#define VTTS_FAMILY_QUICKVC 1
#define VTTS_FAMILY_STABLETTS 2
#define VTTS_FAMILY_T2S 3
#define VTTS_FAMILY_SOVITS 4

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
/* Bytes of device memory and of pinned host memory this process holds through the library right now, over every handle and
 * the handle-free calls.  vtts_destroy gives back everything its handle allocated, so the pair returns to its value from
 * before vtts_create. */
int vtts_debug_live_bytes(uint64_t* device_bytes, uint64_t* pinned_bytes);
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
/* Unit-test hooks for the duration path: each runs the kernels of one stage through the engine's own launch code, on host
 * tensors.  B, lens: utterances packed as the engine packs them (utterance b starts at row offs[b], SEQ_GAP (8) rows between
 * consecutive utterances); every row buffer has `rows` rows (>= the packed utterances), and rows outside the utterances keep
 * what the caller wrote in every in/out buffer.  Malformed arguments return VTTS_ERR_INVALID before anything is launched.
 *
 * vtts_debug_dds: the three DDSConv layers (dilations 1, k, k^2; dds_layer_kernel) of `stack` of the loaded model, launched
 * as dds_stack launches them:
 *   "dp.convs"              x fp32 [rows][dp_filter_channels]; x0 and cond NULL
 *   "dp.flows.<i>.convs"    the ConvFlow at the reference's module index i = 2n - 1 (n = 2 .. dp_n_flows), its front
 *                           pre(x0) + cond fused into layer 0: x0 fp32 [rows], cond fp32 [rows][dp_filter_channels]; x NULL
 *   y                       out (in/out) fp32 [3][rows][dp_filter_channels]: the output of each layer (layer i > 0 reads
 *                           layer i - 1's); y[2] is the stack's result */
int vtts_debug_dds(vtts_handle h, const char* stack, int B, const int* lens, size_t rows, const float* x, const float* x0,
                   const float* cond, float* y);
/* vtts_debug_spline: spline_inverse_kernel on params fp32 [rows][ldh] (widths | heights | interior derivatives, 3 * nb - 1
 * used, unscaled as the ConvFlow's proj writes them) and x1 fp32 [rows] (in place), with the engine's dp_num_bins (nb),
 * dp_tail_bound and sqrt(dp_filter_channels). */
int vtts_debug_spline(vtts_handle h, int B, const int* lens, size_t rows, const float* params, int ldh, float* x1);
/* vtts_debug_durations: duration_kernel, then sample_prior_kernel, as phase 1 and phase 2 run them.
 *   z [rows]                    the flows' output x1 channel; logw = (z - m) * exp(-logs) with the model's ElementwiseAffine
 *   length_scale, frame_cap     frame_cap > 0: the frame count a speculative second phase is sized for (0: none)
 *   stats [rows][2I], eps [B][I][eps_ld], noise_scale    the prior: z_p = m + eps * exp(logs) * noise_scale (I = inter_channels)
 *   wceil, cum [rows]           out (in/out) int: ceil durations and their inclusive scan
 *   ylen, ylen_real [B]         out: the device frame lengths (capped at frame_cap) and the true ones
 *   frm_off [B + 1]             out: the device frame offsets (capped layout)
 *   published [2B + 1]          out: the lengths and offsets the host reads (uncapped)
 *   z_p [frame_rows][I], frame_token [frame_rows]    out (in/out): the prior sample and token of every frame
 * Durations summing past INT32_MAX frames (an utterance, or the batch's frame rows) return VTTS_ERR_INVALID after the
 * duration kernel, as vtts_durations does; frame_rows or eps_ld too small return VTTS_ERR_CAPACITY. */
int vtts_debug_durations(vtts_handle h, int B, const int* lens, size_t rows, const float* z, float length_scale, int frame_cap,
                         const float* stats, const float* eps, int64_t eps_ld, float noise_scale, int32_t* wceil, int32_t* cum,
                         int32_t* ylen, int32_t* ylen_real, int32_t* frm_off, int32_t* published, size_t frame_rows, float* z_p,
                         int32_t* frame_token);
/* vtts_debug_stt_durations (StableTTS engines with a text encoder): stt_dur_kernel, stt_expand_kernel, stt_pause_fill_kernel.
 *   mu_dp [rows][dur_channels], pause [rows], length_scale      the duration rule's inputs (pauses as given, unchecked)
 *   x [rows][cond_channels], mu_mel [rows][noise_channels]      token rows expanded to frames (mu_mel may be NULL without prior)
 *   denormalise                 prior rows times mel_std plus mel_mean
 *   dur, first [rows] int, logw [rows], ylen [B]     out (dur, first, logw in/out): durations, first frames, pre-rounding values
 *   mu [frame_rows][cond_channels], pau [frame_rows], prior [frame_rows][noise_channels] or NULL    out (in/out): the expansion
 *   mel [frame_rows][noise_channels]    in/out: the pause fill runs on it
 * Frame rows are packed from ylen as the mel phase packs them; frame_rows too small returns VTTS_ERR_CAPACITY. */
int vtts_debug_stt_durations(vtts_handle h, int B, const int* lens, size_t rows, const float* mu_dp, const float* pause,
                             float length_scale, const float* x, const float* mu_mel, int denormalise, int32_t* dur, int32_t* first,
                             int32_t* ylen, float* logw, size_t frame_rows, float* mu, float* pau, float* prior, float* mel);
/* Unit-test hooks of the spectral kernels, with the packing and in/out rules of the duration hooks above.
 * vtts_debug_front_end: the front end of vtts_convert / vtts_align / vtts_speaker_embedding (clip lengths checked and framed
 * as they are, staged with NaN behind every clip) on wav [B][ld] (from_spec 0) or features [B][spec_channels][ld] (1):
 * frames [B] out, mag [rows][filter_length/2+1] (in/out, mel engines' waveform input only, else NULL) and feat [rows][spec_pad
 * (spec_channels rounded up to 16, n_mel_channels for QuickVC)] (in/out), rows packed from the frame counts. */
int vtts_debug_front_end(vtts_handle h, int from_spec, const float* in, const int64_t* lengths, int B, int64_t ld, int32_t* frames,
                         size_t rows, float* mag, float* feat);
/* vtts_debug_istft: istft_pqmf_kernel as the decoders launch it, on conv_post rows post [rows][subbands * (istft_n_fft + 2)]
 * of B utterances of lens[b] frames, packed from row `first` (utterance b: up_total * lens[b] + 1 rows from up_total * offs[b]
 * + b) -> wav [n_wav] (in/out; utterance b: hop * lens[b] samples from hop * offs[b]). */
int vtts_debug_istft(vtts_handle h, int B, const int* lens, int first, size_t rows, const float* post, size_t n_wav, float* wav);
/* vtts_debug_mrf_mean: the MRF mean of n (1..3) resblock outputs x [n][rows][C] (utterance b: rmul * lens[b] rows from rmul *
 * offs[b]).  use_tc 0: mrf_mean_kernel over all rows -> out [rows][C]; hi / lo NULL.  use_tc 1: mrf_mean_planes_kernel ->
 * split-bf16 planes hi / lo [plane_rows][C] (in/out) of lrelu(mean, last ? 0.01 : 0.1), with `last` the reflect row at
 * row rmul * offs[b] + b, and the mean into out [rows][C] (in/out) unless NULL. */
int vtts_debug_mrf_mean(vtts_handle h, int use_tc, int B, const int* lens, int rmul, int C, int n, size_t rows, const float* x,
                        int last, float* out, size_t plane_rows, uint16_t* hi, uint16_t* lo);
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
 *                on its own samples; needs wav_lengths[b] >= max(pad + 1, hop_length) (385 samples for the reference configuration)
 *   noise_scale  scales the posterior's eps (the reference uses 1); 0 gives z = m
 *   noise_q      float [B, inter_channels, q_ld] replaces torch.randn_like at models.py:841 (columns < frames[b] read), or
 *                NULL -> Philox(seed)
 *   out_wav      out float [B, out_ld]: clip b gets hop * out_frames[b] samples
 *   out_frames   out int64 [B]
 * Host pointers, atomic on the handle.  VTTS_ERR_INVALID: the blob has no enc_q, n_speakers <= 1, a speaker id out of range,
 * a clip too short for the reflect padding and one frame, or an odd flow_n_flows (the Flip folding of the packed flow is only valid for
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
 * model, a clip too short for the reflect padding and one frame, t_x < 1, t_x > frames (no monotonic path exists) or t_x > 2048.
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
 *                + 1, pad = (filter_length - hop_length) / 2), and needs wav_lengths[b] >= max(pad + 1, hop_length) (481 samples at
 *                the published configuration)
 *   g_out        out float [B, gin_channels]
 * Host pointers, atomic on the handle.  VTTS_ERR_INVALID: not a QuickVC engine, a clip too short for the reflect padding and one frame. */
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

/* Resampling of recordings to a model's rate, and optional silence trimming: librosa.load(path, sr=...) followed, for
 * QuickVC targets, by librosa.effects.trim(y, top_db=20), as vc/convert.py:65-66 prepares its inputs.  The resampler is
 * scipy.signal.resample_poly(x, up, down) with its defaults (up / down = to_rate / from_rate in lowest terms; a Kaiser
 * (beta 5) windowed-sinc low-pass of 2 * 10 * max(up, down) + 1 taps, cutoff 1 / max(up, down), gain up; zeros outside the
 * clip), not librosa's default soxr_hq: the two differ in filter design, not in kind.  Clip b gives ceil(wav_lengths[b] * up
 * / down) samples; equal rates copy the clip exactly.  Each clip is resampled as if alone: its output is bit-identical in any
 * batch.
 *   wav          float [B, wav_ld], clip b = its first wav_lengths[b] samples, 1 <= wav_lengths[b] <= wav_ld
 *   from_rate, to_rate   in [VTTS_RESAMPLE_MIN_RATE, VTTS_RESAMPLE_MAX_RATE] Hz; the pair's filter must have at most
 *                VTTS_RESAMPLE_MAX_TAPS taps (44 100 <-> 16 000 takes 8 821, 96 000 <-> 22 050 12 801)
 *   trim_top_db  > 0: trim each resampled clip as librosa.effects.trim(y, top_db=trim_top_db) (librosa >= 0.10): frames of 2048
 *                samples at hop 512, centred with zero padding; a frame is kept iff its mean square is above max(1e-10, the
 *                loudest frame's) by more than -trim_top_db dB; the clip keeps [first * 512, min(n, (last + 1) * 512)).
 *                <= 0: no trim.
 *   out          out float [B, out_ld]: clip b's out_lengths[b] samples; the rest of each row is not written.  out_ld must
 *                hold the untrimmed length ceil(wav_lengths[b] * up / down).
 *   out_lengths  out int64 [B]
 *   trim_bounds  out int64 [B, 2] or NULL: [start, end) of each kept part in the untrimmed resampled clip ([0, n) untrimmed)
 * Host pointers, atomic on the handle; serves engines of every model family.  The taps of a rate pair are computed on the
 * host in float64, rounded to fp32 once and kept on the device by the handle.  VTTS_ERR_INVALID: B < 1, a length outside
 * [1, wav_ld], a rate out of range, a pair over the tap cap, a batch whose packed rows exceed
 * VTTS_RESAMPLE_MAX_BATCH_SAMPLES (per clip the larger of its input and output length, plus 8), a clip of digital silence
 * (every frame's mean square <= 1e-10) when trimming.  VTTS_ERR_CAPACITY: out_ld below an untrimmed clip's length. */
#define VTTS_RESAMPLE_MIN_RATE 4000
#define VTTS_RESAMPLE_MAX_RATE 384000
#define VTTS_RESAMPLE_MAX_TAPS 64001
#define VTTS_RESAMPLE_MAX_BATCH_SAMPLES (1LL << 30)
int vtts_resample(vtts_handle h, const float* wav, const int64_t* lengths, int B, int64_t ld, int from_rate, int to_rate,
                  float trim_top_db, float* out, int64_t out_ld, int64_t* out_lengths, int64_t* trim_bounds);

/* StableTTS flow-matching decoder (CFM.forward -> solve_euler -> Decoder, flow_matching.py:33-100,182-194, decoder.py:103-138,
 * as MatchaTTS.synthesise calls it at matcha_tts.py:183): the encoder output expanded to frames and a speaker in, mel out.
 * z = noise * temperature; t_span = 1 - cos(linspace(0, 1, n + 1) pi / 2); n fixed Euler steps x += dt (v_c + s (v_c - v_u))
 * with v_c = estimator(x, mu, t, speaker) and v_u = estimator(x, fake_content, t, fake_speaker) (classifier-free guidance;
 * the reference fixes s = 0.5).  Each utterance is decoded as if alone (the prenet's convs are zero padded at its own ends),
 * and its mel is bit-identical in any batch.  One call is one enqueue: no host wait between the steps.
 *   mu           float [B, mu_ld, st_cond], frame-major: utterance b = its first lengths[b] frames, 1 <= lengths[b] <= mu_ld
 *   sid          int64 [B] rows of spk_emb, or NULL when spk_rows is given
 *   spk_rows     float [B, st_spk_dim] speaker embeddings used instead of spk_emb[sid], or NULL
 *   n_timesteps  in [1, VTTS_CFM_MAX_STEPS]
 *   guidance_scale  s >= 0; 0 skips the unconditional branch
 *   noise        float [B, noise_ld, st_noise] frame-major, standing in for torch.randn (flow_matching.py:52), or NULL for
 *                Philox(seed); with noise given, seed is not read
 *   mel_out      out float [B, mel_ld, st_noise] frame-major: utterance b's lengths[b] frames, the rest of each row is not written
 *   denormalise  != 0: mel * mel_std + mel_mean (matcha_tts.py:205), else the normalised mel of the last Euler step
 * Host pointers, atomic on the handle; graphed per (batch, frame bucket, n_timesteps, s == 0, noise / speaker input kind).
 * Runs on the fp32 FFMA pipe in precision modes 0, 1 and 3; in mode 2 the estimator's convs whose widths are multiples of 64
 * and its attention run on split-bf16 wgmma (in_proj, final_proj and the Euler update stay fp32), an utterance's mel still the
 * same alone and in any batch.  VTTS_ERR_INVALID: not a StableTTS engine, B < 1, a length outside
 * [1, mu_ld], n_timesteps out of range, a temperature or guidance scale that is not finite (or s < 0), a speaker id outside
 * [0, st_n_spks), neither sid nor spk_rows.  VTTS_ERR_CAPACITY: mel_ld or noise_ld below the longest utterance.
 * After a call with bit0 of vtts_debug_flags set, vtts_debug_read gives "st_film" [steps][layers][2 hidden], "st_ada"
 * [sequences][layers][6 hidden] (the unconditional sequences after the B conditional ones), "st_cond" (the in_proj operand
 * rows [rows][st_noise + st_hidden]: x after the last step, then cond_proj's output), "st_rope" [max frames][dk / 4] (cos, sin)
 * pairs, and of the first estimator evaluation "st_norm1" (block 0's modulated LayerNorm) and "st_qkv" (block 0's q, k
 * after the rotary embedding, and v), rows [rows][hidden] and [rows][3 hidden].  In precision mode 2 also, of block 0 at step
 * 0, each plane-writing kernel's input and output rows: "tc_norm_in", "tc_qkv_in" (before the rotary embedding),
 * "tc_silu_in", "tc_silu", "tc_gate_x", "tc_gate_y", "tc_gate" (fp32 rows), and the planes of "tc_norm", "tc_qkv",
 * "tc_silu" and "tc_gate" as "<name>_hi" / "<name>_lo" (bf16 bit patterns, two per float), for the kernels whose consumer
 * runs on the tensor cores. */
#define VTTS_CFM_MAX_STEPS 64
int vtts_cfm_decode(vtts_handle h, const float* mu, const int64_t* lengths, int B, int64_t mu_ld, const int64_t* sid,
                    const float* spk_rows, int n_timesteps, float temperature, float guidance_scale, const float* noise,
                    int64_t noise_ld, uint64_t seed, float* mel_out, int64_t mel_ld, int denormalise);

/* StableTTS text-to-mel (MatchaTTS.synthesise, training/stabletts/matcha/models/matcha_tts.py:93-211; the graph
 * matcha/onnx/export.py exports without a vocoder): multistream ids, BERT features and pause durations in, durations and mel
 * out.  x = (emb(ids[0]) sqrt(160) | punc_emb(ids[1..4]) sqrt(16) | bert_proj(bert)); dp_encoder(x, dur_spk_emb[sid]) -> 50
 * channels; a token's duration is the sum of their sigmoids, or its pause where that is not 0, times length_scale, rounded
 * half to even, at least 1; mu_y = x expanded by the durations; the decoder of vtts_cfm_decode refines it; every frame of a
 * token with a pause > 0 takes the mel of the utterance's frame 0.
 * Each utterance is processed as if alone: its own frame 0 is its silence frame (the reference, called with one utterance,
 * takes utterance 0's), and the decoder's unmasked stages (noise, cond_proj, in_proj) run on its own frame count rounded up
 * to a multiple of 4, as synthesise pads it (matcha_tts.py:162-165).  Durations and mel are bit-identical in any batch.
 *   ids          int64 [B, st_streams, t_max], each in [0, st_n_vocab); utterance b = the first id_lengths[b] columns
 *   bert         float [B, t_max, st_bert_dim], token-major
 *   pause        float [B, t_max] (phone_duration_extra, frames before length_scale; 0: predict), or NULL for none
 *   sid          int64 [B] rows of spk_emb and dur_spk_emb
 *   noise        float [B, noise_ld, st_noise] frame-major, standing in for torch.randn over the padded frame axis
 *                (flow_matching.py:54): ceil4(frames) rows per utterance are read; or NULL for Philox(seed)
 *   mel_out      out float [B, mel_ld, st_noise] frame-major, mel_lengths[b] frames of utterance b; the rest is not written
 *   mel_lengths  out int64 [B]
 *   durations    out int32 [B, t_max] frames of every token (0 past id_lengths[b]), or NULL
 *   prior_out    out float [B, mel_ld, st_noise]: the mel encoder's output expanded to frames (encoder_outputs; mel_enc with
 *                denormalise), or NULL: the mel encoder then does not run
 *   denormalise  != 0: mel * mel_std + mel_mean
 * Two enqueues with one host wait between them for the frame counts: the text phase is graphed per (batch, token bucket),
 * the mel phase per (batch, token and frame buckets, n_timesteps, s == 0, noise kind).  The text phase is fp32 FFMA in every
 * precision mode, so durations and frame counts do not depend on it; the mel phase is as in vtts_cfm_decode (mode 2: on
 * the tensor cores).
 * VTTS_ERR_INVALID: not a StableTTS engine or a decoder-only blob, B < 1, t_max outside [1, VTTS_ST_MAX_TOKENS], a length
 * outside [1, t_max], an id or speaker out of range, a pause outside [0, VTTS_ST_MAX_TOKEN_FRAMES], length_scale outside
 * (0, 100], the sampling arguments as vtts_cfm_decode.  VTTS_ERR_CAPACITY, returned after the text phase with mel_lengths
 * filled in: mel_ld below the longest utterance, or noise_ld below it rounded up to a multiple of 4.
 * After a call, vtts_debug_read gives "st_tok_x" (the token rows x [tokens][st_cond]), "st_mu_dp" [tokens][st_dur_channels],
 * "st_logw" [tokens] (durations before rounding) and "st_mu" (the decoder's mu rows [rows][st_cond], packed by padded frame
 * count, the unconditional sequences after the conditional ones). */
#define VTTS_ST_MAX_TOKENS 16384
#define VTTS_ST_MAX_TOKEN_FRAMES 4096
int vtts_stabletts_synthesise(vtts_handle h, const int64_t* ids, const int64_t* id_lengths, int B, int64_t t_max, const float* bert,
                              const float* pause, const int64_t* sid, int n_timesteps, float temperature, float length_scale,
                              float guidance_scale, const float* noise, int64_t noise_ld, uint64_t seed, float* mel_out, int64_t mel_ld,
                              int64_t* mel_lengths, int32_t* durations, float* prior_out, int denormalise);

/* StableTTS vocoder: the HiFi-GAN Generator of training/stabletts/matcha/hifigan/models.py:148-206 (conv_pre, n_upsamples x
 * (LeakyReLU 0.1, ConvTranspose1d, mean of the MRF resblocks), LeakyReLU 0.01, conv_post, tanh), as cli.py:65-71 loads it
 * (config v1, weight norm removed) and calls it on a denormalised mel; the reference's clamp(-1, 1) after tanh changes
 * nothing.  Engines whose blob carries dec.* (StableTTS(..., vocoder=...), weights.pack_hifigan), described by the decoder
 * fields of vtts_config: decoder_type 1, resblock_*, upsample_*, upsample_initial_channel, inter_channels = st_noise.
 * Each utterance is vocoded as if alone (zero padding at its own ends, as the reference at batch 1).
 *   mel          float [B, mel_ld, st_noise], frame-major, denormalised; utterance b = its first mel_lengths[b] frames,
 *                1 <= mel_lengths[b] <= mel_ld
 *   wav          out float [B, wav_ld]: utterance b's wav_lengths[b] = hop * mel_lengths[b] samples (hop = the product of the
 *                upsampling rates, 256 for v1); the rest of each row is not written
 * Host pointers, atomic on the handle; graphed per (batch, frame bucket).  Precision 0 runs every conv on the fp32 FFMA pipe
 * in one fixed launch shape: the waveform is bit-identical alone, in any batch, eager and replayed.  Precision >= 1 runs the
 * upsampling convs whose input width is a multiple of 64 and the MRFs of the stages before the last such conv on the
 * split-bf16 tensor cores (for v1: every upsampling conv and the MRFs of stages 1-3); their split-K plans follow the batch,
 * so the waveform is bit-identical eager and replayed but may differ in the last bits between batch shapes.
 * VTTS_ERR_INVALID: not a StableTTS engine, a blob without a vocoder, B < 1, a length outside [1, mel_ld], a batch whose
 * largest vocoder buffer would exceed 2^31 values.  VTTS_ERR_CAPACITY: wav_ld < hop * max(mel_lengths). */
int vtts_hifigan_vocode(vtts_handle h, const float* mel, const int64_t* mel_lengths, int B, int64_t mel_ld, float* wav, int64_t wav_ld,
                        int64_t* wav_lengths);

/* StableTTS text-to-waveform: vtts_stabletts_synthesise followed by vtts_hifigan_vocode on its denormalised mel, in the same two
 * enqueues (the vocoder runs in the mel phase's graph on the mel rows already on the device: no mel round trip, one host wait
 * between the phases as before).  Arguments as vtts_stabletts_synthesise, plus wav [B, wav_ld] and wav_lengths int64 [B]
 * (= hop * mel_lengths) as vtts_hifigan_vocode; mel_out may be NULL (then prior_out must be NULL too).  Each utterance is
 * vocoded over its own frame count, not its padded extent (matcha_tts.py:184, 207).  Precision 0: wav is bit-identical to
 * vtts_stabletts_synthesise followed by vtts_hifigan_vocode on its denormalised mel.  VTTS_ERR_INVALID also for a blob without
 * a vocoder.  VTTS_ERR_CAPACITY, returned after the text phase with mel_lengths filled in: also wav_ld < hop * max(mel_lengths). */
int vtts_stabletts_synthesise_wav(vtts_handle h, const int64_t* ids, const int64_t* id_lengths, int B, int64_t t_max, const float* bert,
                                  const float* pause, const int64_t* sid, int n_timesteps, float temperature, float length_scale,
                                  float guidance_scale, const float* noise, int64_t noise_ld, uint64_t seed, float* mel_out, int64_t mel_ld,
                                  int64_t* mel_lengths, int32_t* durations, float* prior_out, int denormalise, float* wav, int64_t wav_ld,
                                  int64_t* wav_lengths);

/* BERT features (the logits of training/stabletts/matcha/onnx/bert-export.py: BertModel(input_ids, attention_mask = 1,
 * token_type_ids = 0).hidden_states[-3], as vosk_tts/synth.py:25-44 runs it on one sentence's word pieces): word + token-type 0
 * + position embeddings and their LayerNorm, then cv_layers post-LN layers.  Each sentence is processed as if alone (its
 * positions count from 0; the reference's all-ones attention mask of one sentence); its rows are bit-identical alone, in any
 * batch, eager and replayed.
 *   ids        int64 [B, ids_ld] WordPiece ids ([CLS] ... [SEP] as the tokenizer gives them); sentence b = its first lengths[b]
 *   out        out float [B, out_ld, cv_hidden]: the last layer's rows of sentence b, zeros after them
 * Host pointers, atomic on the handle; graphed per (batch, longest-sentence bucket, row bucket).  Precision 0 runs on the fp32
 * FFMA pipe in one fixed launch shape; modes >= 1 run the GEMMs on the split-bf16 tensor cores without split-K and the
 * attention on attn_tc_kernel (the ContentVec path).  VTTS_ERR_INVALID: not a StableTTS engine, a blob without bt.*, B < 1, a
 * length outside [1, ids_ld] or above the position table's rows (the reference's lookup fails there too), an id
 * outside the word table.  VTTS_ERR_CAPACITY: out_ld below a sentence's length. */
int vtts_bert_features(vtts_handle h, const int64_t* ids, const int64_t* lengths, int B, int64_t ids_ld, float* out, int64_t out_ld);

/* StableTTS text-to-waveform from word pieces: vtts_stabletts_synthesise_wav with each token's BERT row computed and gathered on
 * the device (what vosk_tts/synth.py:25-87 does on the host with get_word_bert and the word index of g2p_multistream*): the
 * text phase's graph runs BERT on every sentence's word pieces (as vtts_bert_features), then copies row bert_rows[b][t] of
 * sentence b's rows to token t.  The [T, bert_dim] features never reach the host.  Arguments as
 * vtts_stabletts_synthesise_wav, with `bert` replaced by
 *   pieces        int64 [B, pieces_ld] WordPiece ids of sentence b ([CLS] ... [SEP]), its first piece_lengths[b]
 *   bert_rows     int32 [B, t_max] the row among sentence b's pieces that token t reads, for t < id_lengths[b]
 * Graphed per (batch, token bucket, BERT's longest-sentence and row buckets).  In every precision mode the outputs are
 * bit-identical to vtts_bert_features, the same gather on the host and vtts_stabletts_synthesise_wav.  VTTS_ERR_INVALID, with
 * nothing launched: also a blob without bt.*, st_bert_dim != cv_hidden, a row outside [0, piece_lengths[b]), and what
 * vtts_bert_features refuses of the pieces. */
int vtts_stabletts_synthesise_pieces_wav(vtts_handle h, const int64_t* ids, const int64_t* id_lengths, int B, int64_t t_max,
                                         const int64_t* pieces, const int64_t* piece_lengths, int64_t pieces_ld, const int32_t* bert_rows,
                                         const float* pause, const int64_t* sid, int n_timesteps, float temperature, float length_scale,
                                         float guidance_scale, const float* noise, int64_t noise_ld, uint64_t seed, float* mel_out,
                                         int64_t mel_ld, int64_t* mel_lengths, int32_t* durations, float* prior_out, int denormalise, float* wav,
                                         int64_t wav_ld, int64_t* wav_lengths);

/* GPT-SoVITS text-to-semantic decoding (Text2SemanticDecoder.infer_panel, training/gpt-sovits/ar/models/t2s_model.py:324-448,
 * with the sampler of ar/models/utils.py:110-161), for a ragged batch of sentences, each decoded as if alone.
 *   ids            int64 [B, ids_ld] phone ids; sentence b = its first lengths[b] (1 <= lengths[b] <= ids_ld, at most the
 *                  position table's rows), every id in [0, rows of t2s.temb)
 *   bert           float [B, ids_ld, 1024] token-major BERT features, or NULL for zeros (bert_proj's bias alone, as the Russian
 *                  voice's get_phones_and_bert gives)
 *   prompts        int64 [B, prompts_ld] semantic tokens of the reference audio with prompt_lengths[b] in [0, prompts_ld], each
 *                  in [0, EOS), or both NULL (no prompt)
 *   top_k >= 1, top_p (applied when < 1), temperature (max(temperature, 1e-5) divides), repetition_penalty > 0 (the reference
 *                  hard-codes 1.35), early_stop_num (-1: none), step_cap (the reference's 1500): an utterance samples at most
 *                  min(step_cap, early_stop_num + 1) tokens (the step limit)
 *   seeds          uint64 [B]: q ~ Exp(1) of entry v at sampling step i drawn by Philox keyed by (seeds[b], i, v); or NULL with
 *   q              float [B, q_ld, V] the reference's q of each sampling step (V = EOS + 1 entries; step 0 reads the first V - 1),
 *                  q_ld >= the step limit; NULL: seeds
 *   tokens         out int64 [B, tokens_ld] (tokens_ld >= prompt length + step limit): y[:, :-1] of each utterance, its prompt
 *                  then the sampled tokens without the last one, n_tokens[b] of them (out int64 [B])
 *   idx            out int64 [B]: the reference's second return value (0 without a prompt, else the sampled count minus 2)
 *   logits         out float [B, logits_ld, V] or NULL: the raw logits of every sampling step below logits_ld (step 0's EOS entry
 *                  included)
 * The [text; prompt] rows are prefilled under infer_panel's prefix mask; then each step samples one token per utterance and
 * runs the layers on it.  An utterance stops, frozen, when its count exceeds early_stop_num, when the argmax of its
 * penalised logits or its sample is EOS, or at step_cap.  The prefill is post_ln_layers: fp32 FFMA in precision
 * mode 0, split-bf16 tensor cores in modes >= 1; the decode steps are fp32 FFMA in every mode.  Each utterance's tokens are
 * the same alone and in any batch.  Host pointers, atomic on the handle.  VTTS_ERR_INVALID, before any launch: not a
 * text-to-semantic engine, B outside [1, 4096], an id or prompt token out of range, a length out of range, a prompt plus the
 * step limit beyond the position table, top_k < 1, a non-finite or non-positive sampling argument, early_stop_num < -1,
 * step_cap outside [1, 2^20], neither seeds nor q, q_ld below the step limit.  VTTS_ERR_CAPACITY: tokens_ld too small. */
int vtts_t2s_decode(vtts_handle h, const int64_t* ids, const int64_t* lengths, int B, int64_t ids_ld, const float* bert,
                    const int64_t* prompts, const int64_t* prompt_lengths, int64_t prompts_ld, int top_k, float top_p, float temperature,
                    float repetition_penalty, int early_stop_num, int step_cap, const uint64_t* seeds, const float* q, int64_t q_ld,
                    int64_t* tokens, int64_t tokens_ld, int64_t* n_tokens, int64_t* idx, float* logits, int64_t logits_ld);
/* Unit-test hook of the text-to-semantic sampler: one t2s_sample_kernel launch, as a decode step launches it, on host rows.
 *   logits [B][V]             one step's logits per row (V = the engine's vocabulary, EOS last)
 *   state (in/out) [B][8]     each row's decode state as the kernel reads it (t2s.cuh T2sSt: P, NY, GEN, STOP, YOFF); YOFF is
 *                             set to b * y_ld
 *   y (in/out) [B][y_ld]      each row's tokens: y[b][0, P + GEN) are its previous tokens (prompt, then sampled), which also
 *                             make its seen bitmap; the sampled token lands at y[b][P + GEN]
 *   top_k .. step_cap         the sampling scalars of vtts_t2s_decode
 *   seeds [B] or q [B][q_ld][V]   the Philox streams, or the caller's Exp(1) draws (row GEN of each)
 *   seen (out) [B][(V + 31) / 32], n_stopped (out): the bitmap after the launch and the rows that stopped in it
 *   raw (in/out) [B][raw_ld][V] or NULL: the raw-logit rows the kernel writes (row GEN, when GEN < raw_ld)
 * VTTS_ERR_INVALID before the launch: not a text-to-semantic engine, B outside [1, 4096], a token outside [0, V), a state out
 * of range, y_ld <= P + GEN, q_ld <= GEN, both or neither of seeds and q, a sampling argument vtts_t2s_decode refuses. */
int vtts_debug_t2s_sample(vtts_handle h, int B, const float* logits, int32_t* state, int32_t* y, int y_ld, int top_k, float top_p,
                          float temperature, float repetition_penalty, int early_stop_num, int step_cap, const uint64_t* seeds,
                          const float* q, int q_ld, uint32_t* seen, int32_t* n_stopped, float* raw, int raw_ld);

/* GPT-SoVITS prompt tokens (model_family 4): a reference recording's semantic codes, as inference_cli.py:176-200 computes
 * them with chinese-hubert-base and SynthesizerTrn.extract_latent (module/models.py:990-993).
 *   wav        float [B, wav_ld] at 16 kHz, clip b = its first wav_lengths[b] samples, already padded by the caller (the
 *              reference appends int(0.3 * the s2 config's sampling_rate) zeros); no normalisation
 *   codes      out int64 [B, codes_ld]: clip b's frames / 2 codes (frames: HuBERT's frames of the clip), -1 after them
 *   out_frames out int64 [B]: the code counts
 * HuBERT runs as vtts_content_units runs ContentVec (fp32 FFMA in mode 0, split-bf16 tensor cores in modes >= 1), with every
 * launch in one shape whatever the batch; ssl_proj (Conv1d(768, 768, 2, stride 2): an odd last frame is dropped), the
 * codebook scores 2 x.E - |E|^2 and their argmax (lowest index on ties) are fp32 FFMA in every mode.  A clip's codes are
 * bit-identical alone and in any batch.  Host pointers, atomic on the handle; one graphed call keyed by batch and
 * sample-length bucket.  VTTS_ERR_INVALID: not a SoVITS engine, B < 1, a clip too short for one HuBERT frame or longer than
 * wav_ld.  VTTS_ERR_CAPACITY: codes_ld below a clip's code count.
 * After a call, vtts_debug_read "sv_proj" is ssl_proj's output rows [pairs][cv_hidden]: clip 0's codes' rows from row 0,
 * clip b's from sum over earlier clips of ceil(frames / 2). */
int vtts_sovits_semantic(vtts_handle h, const float* wav, const int64_t* wav_lengths, int B, int64_t wav_ld, int64_t* codes,
                         int64_t codes_ld, int64_t* out_frames);
/* The same tail on the caller's HuBERT rows (extract_latent of a stored last_hidden_state, as
 * prepare_datasets/3-get-semantic-vosk.py runs it): feats float [B, feats_ld, cv_hidden] frame-major, clip b = its first
 * frames[b] rows (0 allowed).  codes / out_frames as vtts_sovits_semantic. */
int vtts_sovits_latent(vtts_handle h, const float* feats, const int64_t* frames, int B, int64_t feats_ld, int64_t* codes,
                       int64_t codes_ld, int64_t* out_frames);

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
