// engine.cu -- host runtime of the VITS2 inference engine + the C ABI declared in include/vtts.h.
//
// Replaces the one call `self.model.onnx.run(None, args)` (vosk_tts/synth.py:123-126), i.e. the trace
// of SynthesizerTrn.infer (training/vits2/models.py:1679-1704).  The launch sequence below follows that
// function stage by stage; every kernel is in kernels.cuh (fp32 FFMA) or conv_tc.cuh (wgmma).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <thread>
#include <initializer_list>
#include <map>
#include <mutex>
#include <sstream>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/vtts.h"
#include "kernels.cuh"
#include "conv_tc.cuh"
#include "mas.cuh"
#include "attn_tc.cuh"
#include "vc.cuh"
#include "spk.cuh"
#include "contentvec.cuh"
#include "sovits.cuh"
#include "bert.cuh"
#include "dit.cuh"
#include "stabletts.cuh"
#include "hifigan.cuh"
#include "resample.cuh"
#include "owned.cuh"
#include "t2s.cuh"

using namespace vtts;

namespace {
constexpr int CONV_SMEM_MAX = 160 * 1024;   // dynamic shared memory opt-in of conv_kernel<G>


struct Tensor {
  const float* p = nullptr;
  size_t n = 0;
};
struct ConvW {
  const float* w = nullptr;
  const float* b = nullptr;
  int Cin = 0, Cout = 0, k = 0, ldw = 0;
};
struct TcW {     // split-bf16 copy of a conv weight: [k][Cout][Cin]
  const __nv_bfloat16* hi = nullptr;
  const __nv_bfloat16* lo = nullptr;
  const __nv_bfloat16* mid = nullptr;   // third plane of the exact 3-way split (precision mode 3, text encoder)
};
struct Planes {  // split-bf16 activation planes [rows][C]
  __nv_bfloat16* hi = nullptr;
  __nv_bfloat16* lo = nullptr;
  __nv_bfloat16* mid = nullptr;         // third plane (exact 3-way split) or null
  int C = 0;
  long rows = 0;
};
struct TcSpec {  // one problem of a grouped tensor-core conv launch
  Planes in;
  TcW w;
  const float* bias = nullptr;
  int Cin = 0, Cout = 0, k = 1, dil = 1, pad = 0;
  float* y = nullptr; int ldy = 0;
  const float* res = nullptr; int ldr = 0;
  Planes out; float pl_slope = 1.f;
  int out_mul = 1, out_add = 0, in_extra = 0, out_seq_extra = 0;
  int yoff = 0, roff = 0, epi = 0, poff = 0;
  float alpha = 1.f;
  const float* cond = nullptr; int cond_ld = 0;
};
struct LnW {
  const float* g = nullptr;
  const float* b = nullptr;
};
struct EncLayerW {
  ConvW qkv, o, ffn1, ffn2;
  TcW t_qkv, t_o, t_ffn1, t_ffn2;
  LnW ln1, ln2;
  const float* relk = nullptr;
  const float* relv = nullptr;
  int heads = 1;
  // split-bf16 [16][128] tiles of the relative-position tables for the wgmma attention (null: FFMA attention only)
  const __nv_bfloat16 *rk_hi = nullptr, *rk_lo = nullptr, *rv_hi = nullptr, *rv_lo = nullptr;
};
struct DdsW {
  const float *sep_w, *sep_b;
  LnW ln1, ln2;
  ConvW pw;
};
struct CfW {
  const float *pre_w, *pre_b;
  DdsW dds[3];
  ConvW proj;
};
struct FlowW {
  ConvW pre, post;
  EncLayerW tr;
  std::vector<ConvW> in, rsx, rss;
  TcW t_qkv, t_o, t_ffn1, t_ffn2, t_post;
  std::vector<TcW> t_in, t_rsx, t_rss;
};
struct UpW {
  std::vector<ConvW> phase;
  std::vector<TcW> tphase;
  std::vector<int> pad;
};
struct RbW {
  std::vector<ConvW> c1, c2;
  std::vector<TcW> t1, t2;
};

// Launch tuning of the conv and attention kernels.  The engine holds the defaults (from_env); a path that must not depend on
// the batch launches with one of the named fixed shapes below, a copy of the defaults.  Fields are set here and nowhere else.
struct Tuning {
  // FFMA convs (launch_conv): split-K cluster cap, tile target of the split, thread groups per CTA (cap; machine-filling
  // launches; single utterances; k-steps per rank needed to add one, 0 never)
  int conv_max_s = 8, conv_target = 120, conv_max_g = 4, conv_big_g = 1, conv_min_g = 1, conv_auto_g = 4;
  // tensor-core convs (launch_tc)
  int tc_tall = 0, tc_baseoff = 0, tc_dbgskip = 0, tc_bn = 0, tc_mc = 0, tc_split = 0, tc_min_steps = 2, tc_persist = 1,
      tc_persist_min = 1, tc_wmc = 0;
  // attention: query rows per warp (0 auto), the split-KV kernel allowed, wgmma attention where the qkv conv runs on tensor
  // cores (0 never, 1 when throughput bound, 2 always)
  int attn_rows = 0, attn_split = 1, attn_tc_mode = 1;

  static Tuning from_env() {
    Tuning t;
    if (const char* e = getenv("VTTS_CONV_MAXS")) t.conv_max_s = std::max(1, atoi(e));
    if (const char* e = getenv("VTTS_CONV_TARGET")) t.conv_target = std::max(1, atoi(e));
    if (const char* e = getenv("VTTS_CONV_MAXG")) t.conv_max_g = std::max(1, std::min(4, atoi(e)));
    if (const char* e = getenv("VTTS_CONV_BIGG")) t.conv_big_g = std::max(1, std::min(4, atoi(e)));   // thread groups per CTA on machine-filling FFMA launches
    if (const char* e = getenv("VTTS_TC_TALL")) t.tc_tall = atoi(e);
    if (const char* e = getenv("VTTS_TC_BASEOFF")) t.tc_baseoff = atoi(e);
    if (const char* e = getenv("VTTS_TC_BN")) t.tc_bn = atoi(e);
    if (const char* e = getenv("VTTS_TC_MULTICAST")) t.tc_mc = atoi(e);
    if (const char* e = getenv("VTTS_TC_SPLIT")) t.tc_split = atoi(e);
    if (const char* e = getenv("VTTS_TC_MINSTEPS")) t.tc_min_steps = std::max(1, atoi(e));   // k-steps per CTA below which split-K stops
    if (const char* e = getenv("VTTS_TC_PERSIST")) t.tc_persist = atoi(e);                 // 0: one tile per CTA also on machine-filling launches; 2: persistent grid on every launch without split-K (tests)
    if (const char* e = getenv("VTTS_TC_DBGSKIP")) t.tc_dbgskip = atoi(e);                 // timing experiments only (wrong results)
    if (const char* e = getenv("VTTS_TC_WMC")) t.tc_wmc = atoi(e);                         // 1: weight-tile multicast between CTA pairs of persistent launches (measured neutral, off)
    if (const char* e = getenv("VTTS_TC_PERSIST_MIN")) t.tc_persist_min = std::max(1, atoi(e));   // tiles per SM from which the persistent grid is used
    if (const char* e = getenv("VTTS_ATTN_SPLIT")) t.attn_split = atoi(e);       // 0: never use the split-KV attention
    if (const char* e = getenv("VTTS_CONV_AUTOG")) t.conv_auto_g = std::max(0, atoi(e));   // k-steps per rank needed to add thread groups; 0 = never
    if (const char* e = getenv("VTTS_CONV_MING")) t.conv_min_g = std::max(1, std::min(4, atoi(e)));      // 0 auto, 1 off, 2/4/8 cap
    if (const char* e = getenv("VTTS_ATTN_ROWS")) t.attn_rows = atoi(e);
    if (const char* e = getenv("VTTS_ATTN_TC")) t.attn_tc_mode = atoi(e);
    return t;
  }
  // One FFMA conv launch shape whatever the rows (no split-K over a cluster, one thread group): every output is summed in the
  // same order, so a sequence's result does not depend on what it is batched with.  The vocoder in precision mode 0, the
  // QuickVC speaker encoder and both StableTTS phases.
  Tuning fixed_ffma() const {
    Tuning t = *this;
    t.conv_max_s = 1; t.conv_min_g = 1; t.conv_big_g = 1; t.conv_auto_g = 0;
    return t;
  }
  // One attention kernel whatever the rows: the register-blocked FFMA kernel (StableTTS).
  Tuning fixed_attention() const {
    Tuning t = *this;
    t.attn_rows = 4;
    return t;
  }
  // Tensor-core convs without split-K (every output summed by one CTA in one k order, whatever the launch shape) and attention
  // on attn_tc_kernel whenever it takes the layer, unless switched off (ContentVec in precision modes >= 1).
  Tuning fixed_tc() const {
    Tuning t = *this;
    t.tc_split = 1;
    if (t.attn_tc_mode > 0) t.attn_tc_mode = 2;
    return t;
  }
  // vtts_debug_conv's overrides (VTTS_CONV_KEEP: this value)
  Tuning with(const vtts_conv_overrides& ov) const {
    Tuning t = *this;
    auto set = [](int& f, int v) { if (v != VTTS_CONV_KEEP) f = v; };
    set(t.tc_bn, ov.tc_bn); set(t.tc_split, ov.tc_split); set(t.tc_tall, ov.tc_tall); set(t.tc_mc, ov.tc_mc);
    set(t.tc_persist, ov.tc_persist); set(t.tc_wmc, ov.tc_wmc); set(t.tc_min_steps, ov.tc_min_steps); set(t.conv_max_s, ov.conv_max_s);
    set(t.conv_min_g, ov.conv_min_g); set(t.conv_max_g, ov.conv_max_g); set(t.conv_big_g, ov.conv_big_g);
    return t;
  }
  // vtts_debug_attention's kernel selection (VTTS_ATTN_*)
  Tuning with_attention(int kernel) const {
    Tuning t = *this;
    switch (kernel) {
      case VTTS_ATTN_TC: t.attn_tc_mode = 2; break;
      case VTTS_ATTN_SPLIT: t.attn_split = 1; t.attn_rows = 1; break;
      case VTTS_ATTN_R1: t.attn_split = 0; t.attn_rows = 1; break;
      case VTTS_ATTN_R4: t.attn_split = 0; t.attn_rows = 4; break;
      default: break;                               // AUTO / FFMA: the engine's choice
    }
    return t;
  }
};

// The rows a launch runs over: n sequences of at most maxLen rows at the device lengths / offsets the kernels read, the host
// lengths the launch heuristics size for (`sized`: functions of the length buckets only, so that a graph captured for a
// bucket is valid for every call that maps to it), the true host lengths the profiler counts FLOPs with (`real`), and the
// tuning the launches run with.
struct Rows {
  const int *lens, *offs;
  int n, maxLen;
  std::vector<int> sized, real;
  Tuning tune;
};

struct Err {
  int code;
  std::string msg;
};

#define CK(call)                                                                          \
  do {                                                                                    \
    cudaError_t e__ = (call);                                                             \
    if (e__ != cudaSuccess) {                                                             \
      std::ostringstream os__;                                                            \
      os__ << "CUDA error '" << cudaGetErrorString(e__) << "' at " << __FILE__ << ":" << __LINE__ << " in " #call; \
      throw Err{VTTS_ERR_CUDA, os__.str()};                                               \
    }                                                                                     \
  } while (0)

#define REQUIRE(cond, code, text)                     \
  do {                                                \
    if (!(cond)) throw Err{(code), std::string(text)}; \
  } while (0)

}  // namespace

struct vtts_engine {
  // Members are destroyed in reverse order: the stream, declared first, goes last, and the graph execs go before the events.
  Stream stream;
  vtts_config cfg{};
  int device = 0;
  std::mutex mu;
  // The two-phase API (vtts_durations -> vtts_synthesize / vtts_flow) keeps per-handle state between two calls.  A thread
  // that has run vtts_durations owns the handle until its vtts_synthesize / vtts_flow has succeeded (or failed for good);
  // entry points called by OTHER threads wait for that instead of overwriting the pending durations.
  bool two_phase = false;
  std::thread::id owner;
  std::condition_variable cv;
  std::string err;
  uint64_t launches = 0;

  Buf<float> d_blob;
  size_t blob_floats = 0;
  std::unordered_map<std::string, Tensor> tensors;

  // ---- weights (views into d_blob)
  bool has_g = false;
  const float *emb_g = nullptr, *cond_w = nullptr, *cond_b = nullptr, *enc_emb = nullptr, *dp_ea = nullptr;
  const float *istft_basis = nullptr, *pqmf = nullptr;
  const float* istft_w2 = nullptr;      // squared window: the tail divides by the window envelope (torch.istft; QuickVC)
  int condR = 0, r_spk = -1, r_dp = 0, r_flow = 0, r_dec = -1;
  std::vector<EncLayerW> enc;
  ConvW enc_proj, dp_pre, dp_proj, dec_pre, dec_post;
  DdsW dp_dds[3];
  std::vector<CfW> cf;   // index n-2 for n = 2..dp_n_flows
  std::vector<FlowW> flow;
  std::vector<UpW> ups;
  std::vector<RbW> rbs;
  int hop = 0, up_total = 1;
  bool tc = false;                      // precision mode 1: wgmma path for the decoder convs
  TcW tc_pre, tc_post, tc_encproj;
  bool enc_on_tc = false;               // precision modes 2 / 3: the text encoder's convs on wgmma as well
  bool enc_three = false;               // mode 3: with the exact 3-way operand split
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  EncodeFn encode_tiled = nullptr;
  Buf<__nv_bfloat16> pl_pool[128];            // plane buffers (hi/lo pairs), indexed by the decoder code
  unsigned long long* tc_dbg = nullptr;     // device stamps buffer (microbench)
  TcBatch tc_batch;                         // launch_tc's parameter block (calls on one handle are serialised by `mu`)
  double tc_prof_flops = 0.0;
  uint64_t tc_prof_launches = 0;
  std::vector<Event> tc_prof_ev;
  size_t tc_prof_used = 0;

  // ---- per-call state
  // Ttok / maxTok / Tfrm / maxFrm are the BUCKETED row counts that size buffers, grids, tensor maps and captured graphs
  // (== the real ones with VTTS_BUCKETS=0); the kernels themselves read the true lengths / offsets from device memory.
  // real_* hold the true values for host-side copies; v_*_len are virtual per-utterance lengths (functions of the buckets
  // only) for the launch heuristics, so that a graph captured for a bucket is valid for every call that maps to it.
  int B = 0, Ttok = 0, maxTok = 0, Tfrm = 0, maxFrm = 0;
  int real_Ttok = 0, real_maxTok = 0, real_Tfrm = 0, real_maxFrm = 0;
  std::vector<int> v_tok_len, v_frm_len;
  bool use_buckets = true;
  // Speculative second phase (single utterances): the frame count is data dependent, but the kernels read it from device
  // memory and the host only needs an upper bound -- the length bucket -- to size grids and pick the graph.  The bound is
  // predicted from the frames-per-(token x length_scale) ratio of recent calls, phase 2 is enqueued for that bucket right
  // behind phase 1 WITHOUT the host waiting for the lengths, and repeated with the right bucket in the rare case the
  // prediction was too small.  A whole utterance is then two graph launches and one synchronisation; the phase-1 ->
  // host -> phase-2 round trip (~50 us, and the part of a step most exposed to host jitter) is gone.
  // OFF by default (VTTS_SPEC=1): measured on never-seen utterances with random speakers, whose frames-per-token ratio is
  // heavy tailed (1.3 .. 4), the predicted bucket is usually far too large (the predictor must cover the recent maximum or pay a
  // repeat), the launch heuristics then size split-K / tiles / attention for 3x the rows, and the GPU part of a call grows
  // from 1.7 to 2.5 ms -- while the round trip it removes was already hidden behind the prior projection (value: 1.665 vs
  // 1.666 ms with and without).  It only pays for repeated or very regular texts.
  bool use_spec = false;
  float spec_hist[16] = {};
  int spec_n = 0;
  float spec_ratio = 0.f;
  uint64_t spec_hits = 0, spec_misses = 0;
  double spec_units() const { return (double)real_maxTok * (double)std::max(0.05f, scales[1]); }
  double host_us[8] = {};             // host-side wall clock of the last vtts_infer call: [0] phase-1 enqueue, [1] phase-2 enqueue
                                      //   (+ copy-back enqueue), [2] wait for the stream, [3] copy-out, [4] total, [5] 1 = speculative hit, 2 = miss
  int spec_cap = 0;                   // length bucket of the speculative second phase of the current call (0: not speculating)
  float spec_margin = 1.08f;
  int spec_predict() const { return (int)std::ceil((double)spec_ratio * spec_margin * spec_units()) + 8; }
  void spec_learn() {
    spec_hist[spec_n++ % 16] = (float)((double)real_maxFrm / spec_units());
    float m = 0.f;
    for (int i = 0; i < std::min(spec_n, 16); ++i) m = std::max(m, spec_hist[i]);
    spec_ratio = m;
  }
  // Row offsets of items packed as the engine's rows (tokens or frames): item b starts at off[b], SEQ_GAP rows between
  // items, off[n] the total.  frame_offsets_kernel is the device's copy of this rule.
  static void pack_rows(const std::vector<int>& len, std::vector<int>& off) {
    const size_t n = len.size();
    off.assign(n + 1, 0);
    for (size_t b = 0; b < n; ++b) off[b + 1] = off[b] + len[b] + (b + 1 < n ? SEQ_GAP : 0);
  }
  void pack_frames(const std::vector<int>& frames) {      // host-side frame shape of a call on recordings
    h_frm_len = frames;
    pack_rows(h_frm_len, h_frm_off);
    set_frame_shape();
  }
  void assume_frames(int frames) {      // host-side frame shape from a prediction (B == 1)
    h_frm_len.assign(1, frames);
    h_frm_off = {0, frames};
    set_frame_shape();
  }
  bool read_published_lengths() {       // what frame_offsets_kernel wrote into mapped host memory; false: not there (yet)
    if (!map.p || map.p[0] != call_seq) return false;
    h_frm_len.assign(map.p + 1, map.p + 1 + B);
    h_frm_off.assign(map.p + 1 + B, map.p + 1 + 2 * B + 1);
    check_frame_lengths(h_frm_len.data(), h_frm_off[B], B);
    return true;
  }
  // The frame lengths duration_kernel leaves: -1 for an utterance whose durations sum past INT32_MAX frames, and a total
  // offset of -1 for a batch whose frame rows do not fit an int (the engine indexes frame rows with int).
  static void check_frame_lengths(const int* len, int total, int n) {
    for (int b = 0; b < n; ++b) REQUIRE(len[b] >= 1, VTTS_ERR_INVALID, "an utterance's durations sum past INT32_MAX frames");
    REQUIRE(total >= 0, VTTS_ERR_INVALID, "the batch's durations sum past INT32_MAX frames");
  }
  int eps_dp_ld = 0;                 // row pitch of the duration-predictor noise the phase-1 kernels read
  static int bucket_tok(int n) { return n <= 256 ? (n + 15) / 16 * 16 : (n + 63) / 64 * 64; }
  static int bucket_frm(int n) {
    return n <= 256 ? (n + 31) / 32 * 32 : (n <= 1024 ? (n + 63) / 64 * 64 : (n <= 4096 ? (n + 127) / 128 * 128 : (n + 511) / 512 * 512));
  }
  static void virtual_lens(std::vector<int>& v, int nB, int total_cap, int max_cap) {
    const int per = std::max(1, std::min(max_cap, (total_cap - (nB - 1) * SEQ_GAP + nB - 1) / nB));
    v.assign(nB, per);
  }
  void set_token_shape() {      // from h_tok_len / h_tok_off (real)
    real_Ttok = h_tok_off[B];
    real_maxTok = 0;
    for (int b = 0; b < B; ++b) real_maxTok = std::max(real_maxTok, h_tok_len[b]);
    if (use_buckets) {
      maxTok = bucket_tok(real_maxTok);
      Ttok = B == 1 ? maxTok : (real_Ttok + 63) / 64 * 64;
    } else { maxTok = real_maxTok; Ttok = real_Ttok; }
    virtual_lens(v_tok_len, B, Ttok, maxTok);
    if (!use_buckets) v_tok_len = h_tok_len;
  }
  void set_frame_shape() {      // from h_frm_len / h_frm_off (real)
    real_Tfrm = h_frm_off[B];
    real_maxFrm = 0;
    for (int b = 0; b < B; ++b) real_maxFrm = std::max(real_maxFrm, h_frm_len[b]);
    if (use_buckets) {
      maxFrm = bucket_frm(real_maxFrm);
      Tfrm = B == 1 ? std::max(maxFrm, real_Tfrm) : (real_Tfrm <= 8192 ? (real_Tfrm + 255) / 256 * 256 : (real_Tfrm + 1023) / 1024 * 1024);
    } else { maxFrm = real_maxFrm; Tfrm = real_Tfrm; }
    virtual_lens(v_frm_len, B, Tfrm, maxFrm);
    if (!use_buckets) v_frm_len = h_frm_len;
  }
  // the rows of the current call shape, at the engine's tuning
  Rows tok_rows() const { return Rows{d_tok_len.p, d_tok_off.p, B, maxTok, v_tok_len, h_tok_len, tune}; }
  Rows frm_rows() const { return Rows{d_frm_len.p, d_frm_off.p, B, maxFrm, v_frm_len, h_frm_len, tune}; }
  // plane buffers whose rows behind each utterance must be zeroed for this phase (see zero_tails_kernel)
  TailList tail;
  bool collecting = false;
  void begin_planes() { tail.n = 0; collecting = true; }
  void flush_tails(const int* lens, const int* offs) {
    collecting = false;
    if (tail.n == 0) return;
    klaunch(zero_tails_kernel, dim3(tail.n, B), dim3(128), (size_t)0, tail, lens, offs, B);
    CK(cudaGetLastError());
    ++launches;
  }
  bool have_durations = false;
  float scales[3] = {0.f, 1.f, 0.f};
  uint64_t seed = 0;
  std::vector<int> h_tok_len, h_tok_off, h_frm_len, h_frm_off;

  // ---- workspace
  Buf<int> d_ids, d_tok_len, d_tok_off, d_sid, d_wceil, d_cum, d_frm_len, d_frm_off, d_ftok, d_done_ctr, d_frm_len_real;
  Buf<float> d_condv, d_x, d_xb, d_qkv, d_ao, d_y, d_ffh, d_stats, d_dA, d_dB, d_dx, d_spl, d_za, d_zb, d_eps_dp;
  Buf<float> d_z, d_h, d_h1, d_wx, d_acts, d_skip, d_fqkv, d_fao, d_fy, d_ffh2, d_eps_z, d_d0, d_post, d_wav;
  std::vector<Buf<float>> d_stage;               // X_i
  std::vector<std::vector<Buf<float>>> d_xj, d_tmp;
  // per-launch profiling of the conv kernel family (bench.py roofline): event pairs around each launch
  bool profiling = false;
  std::vector<Event> prof_ev;
  size_t prof_used = 0;
  double prof_flops = 0.0;
  uint64_t prof_launches = 0;
  Buf<unsigned long long> d_tl;                  // vtts_timeline's counter and (source line, ns) pairs
  Buf<float> d_zp_dbg;                           // copy of z_p kept when debug_flags & 1
  int debug_flags = 0;
  Buf<float> d_prm;                              // per-call scalars (see kernels.cuh prm_seed)
  MappedBuf<int> map;                            // mapped pinned host memory: [0] sequence flag, lengths, offsets
  int call_seq = 0;
  bool use_poll = true;
  Event ev[8];
  Stream side[3];                          // branch streams of the decoder's independent resblock chains (forked / joined with events)
  Event ev_fork, ev_join[3];
  // CUDA graphs: a call shape seen before is captured once and replayed (launch-bound at batch 1)
  struct GraphEntry { GraphExec exec; uint64_t gen = 0; uint64_t used = 0; uint64_t nlaunch = 0; int seen = 0; };
  std::map<std::vector<long long>, GraphEntry> graphs;
  uint64_t ws_gen = 0, graph_clock = 0, graph_replays = 0;
  bool capture_on_first = true;
  bool capturing = false, use_graphs = true, last_graphed = false, use_pdl = true;    // programmatic dependent launch (VTTS_PDL=0 turns it off)
  Tuning tune;                             // the launch tuning of every path without a fixed launch shape
  int n_sm = 132;
  // shape of the last dense conv launch (vtts_debug_conv) and, while log_conv is set, of every one (vtts_debug_conv_log)
  vtts_conv_report last_conv{};
  vtts_attn_report last_attn{};               // the last attention launch (vtts_debug_attention)
  bool log_conv = false;
  std::vector<vtts_conv_report> conv_log;
  void note_conv(const vtts_conv_report& r) {
    last_conv = r;
    if (log_conv) conv_log.push_back(r);
  }
  int tc_cluster_cap[2][3] = {{0, 0, 0}, {0, 0, 0}};   // co-resident clusters of 2/4/8 conv_tc CTAs, [BN 64/128][log2(S)-1]   // multicast measured slower (see DESIGN.md 4.2)
  int mrf_heavy_first = 1;
  int mrf_branch = 0;                      // VTTS_MRF_BRANCH=1: one stream per resblock chain (measured slower: 1.74 vs 1.62 ms)
  float stage_ms[8] = {};
  bool ev_valid = false;

  // -------------------------------------------------------------------------------------------
  template <typename T, Mem M>
  T* ensure(Buf<T, M>& b, size_t n) {
    if (n > b.cap) {
      REQUIRE(!capturing, VTTS_ERR_STATE, M == Mem::Device ? "workspace growth during graph capture" : "staging growth during graph capture");
      if (M == Mem::Pinned && b.p) CK(cudaStreamSynchronize(stream));   // copies staged through the old buffer may still be in flight
      CK(b.grow(n));
      ++ws_gen;                                // captured graphs hold the old pointers
    }
    return b.p;
  }

  // Pinned staging of one kind of call input or output: a pinned block and the ordered fields a call copies to or from it,
  // each from or to one engine buffer (n elements of the buffer from element `at`).  A call lists its fields (begin, add),
  // sizes the block once (commit; for an input kind the destinations as well, while a readback never grows its sources), and
  // enqueues the copies where its enqueue runs them, one cudaMemcpyAsync per field in field order, to or from the buffer as
  // it is at that moment: upload after the host has filled the fields, download before the host reads them.  The host
  // names a field by its buffer (host).  A field may reserve room for more elements than it copies, so that a block sized
  // for a length bucket does not grow with every new length.
  // A replayed graph copies to or from the pinned addresses it captured, so the layout of a call must follow from its graph
  // key alone.  It does by construction: each field starts at the first 64-byte boundary behind the one before, so the
  // layout is a function of the field sizes, and those are the sizes of the copies the graph holds.
  struct Staging {
    struct Field { void* buf; size_t off, at, n, bytes, room; void* (*dev)(vtts_engine&, void* buf, size_t at, size_t n, bool grow); };
    vtts_engine* e = nullptr;
    bool readback = false;                       // copied from its buffers (vtts_create sets it: a kind goes one way)
    PinnedBuf<char> pin;
    std::vector<Field> fields;
    size_t end() const { return fields.empty() ? 0 : fields.back().off + fields.back().room; }
    void begin() { fields.clear(); }
    template <typename T>
    void add(Buf<T>& buf, size_t n, size_t at = 0, size_t room = 0) {
      fields.push_back({&buf, (end() + 63) / 64 * 64, at, n, n * sizeof(T), std::max(n, room) * sizeof(T),
                        [](vtts_engine& h, void* b, size_t at, size_t k, bool grow) -> void* {
                          Buf<T>& d = *static_cast<Buf<T>*>(b);
                          REQUIRE(grow || d.cap >= at + k, VTTS_ERR_STATE, "a readback reads past the end of its source buffer");
                          return (grow ? h.ensure(d, at + k) : d.p) + at;
                        }});
    }
    void commit() {
      e->ensure(pin, end());
      if (!readback)
        for (const Field& f : fields) f.dev(*e, f.buf, f.at, f.n, true);
    }
    template <typename T>
    T* host(const Buf<T>& buf) {
      for (const Field& f : fields)
        if (f.buf == &buf) return reinterpret_cast<T*>(pin.p + f.off);
      throw Err{VTTS_ERR_STATE, "a staged field was named that the call does not copy"};
    }
    void upload() {
      for (const Field& f : fields)
        CK(cudaMemcpyAsync(f.dev(*e, f.buf, f.at, f.n, true), pin.p + f.off, f.bytes, cudaMemcpyHostToDevice, e->stream));
    }
    void download() {
      for (const Field& f : fields)
        CK(cudaMemcpyAsync(pin.p + f.off, f.dev(*e, f.buf, f.at, f.n, false), f.bytes, cudaMemcpyDeviceToHost, e->stream));
    }
    // outside a graph: download, mark the end of the call's device work (ev[7], read by collect_timings) and wait for it
    void download_and_wait() {
      download();
      CK(cudaEventRecord(e->ev[7], e->stream));
      CK(cudaStreamSynchronize(e->stream));
    }
  };
  // One staging per kind of input or output; what one call holds at the same time is in different kinds.
  enum StagingKind {
    STG_TOKENS,       // token lengths, offsets and ids, and phase 1's scalars, speaker ids and noise (TTS phase 1, alignment)
    STG_NOISE_Z,      // phase 2's noise_z
    STG_CLIPS,        // calls on recordings (conversion, alignment, speaker embedding, QuickVC conversion)
    STG_CONTENTVEC, STG_BERT, STG_ST_TEXT, STG_ST_PIECES, STG_ST_MEL, STG_VOCODER, STG_RESAMPLE, STG_T2S,
    STG_SPK_SLICES,   // the speaker encoder's slice table
    STG_CHUNK,        // the rows of vtts_decode_chunk
    STG_SOVITS,       // the SoVITS tail's row tables, and the caller's HuBERT rows (vtts_sovits_latent)
    STG_OUT,          // readbacks from here on: a call's outputs
    STG_LENGTHS,      // phase 1's frame lengths and offsets without polling (copied inside its graph)
    STG_T2S_STOP0, STG_T2S_STOP1,   // T2S's count of stopped utterances after an even / odd chunk (two chunks in flight)
    STG_ST_DURATIONS, // the StableTTS text phase's d_sttd (copied inside its graph)
    STG_TRIM,         // the resampler's frame energies
    STG_KINDS
  };
  Staging stg[STG_KINDS];                        // (vtts_create points each at its engine)

  // Runs `enqueue` (which only enqueues work on `stream`) eagerly the first time a shape key is seen -- that run also
  // performs every workspace growth -- and right behind it records the same work into a CUDA graph (capture only, no second
  // execution), so that the SECOND call of a bucket already replays.  The key is the full tuple of everything the
  // enqueued work depends on besides device-resident data (phase tag, batch, length buckets, noise mode, raw pointers of
  // the *_dev entry points): entries are compared on the tuple itself, so there is no hash collision to replay a wrong
  // graph on.  The cache is bounded (LRU, checked on every insertion).
  static constexpr size_t GRAPH_CACHE_MAX = 48;
  // phase tag, the first element of every key
  enum GraphTag : long long {
    TAG_PHASE1 = 0x11, TAG_PHASE2 = 0x22, TAG_PHASE1_DEV = 0x33, TAG_PHASE2_DEV = 0x44, TAG_CONVERT = 0x55, TAG_ALIGN = 0x66,
    TAG_QUICKVC = 0x77, TAG_QUICKVC_WAV = 0x78, TAG_CONTENTVEC = 0xC7, TAG_CFM = 0xCF, TAG_ST_TEXT = 0xD1, TAG_ST_MEL = 0xD2, TAG_HIFIGAN = 0xD3,
    TAG_BERT = 0xD4, TAG_ST_TEXT_PIECES = 0xD5, TAG_T2S = 0xE1, TAG_SOVITS = 0xE2, TAG_SOVITS_LATENT = 0xE3
  };
  template <typename Fn>
  void run_graphed(std::initializer_list<long long> key_il, Fn&& enqueue) {
    last_graphed = false;
    if (!use_graphs || profiling || debug_flags) { enqueue(); return; }
    const std::vector<long long> key(key_il);
    auto it = graphs.find(key);
    if (it == graphs.end()) {
      if (graphs.size() >= GRAPH_CACHE_MAX) {       // evict the least recently used entry before inserting
        auto old = graphs.begin();
        for (auto k = graphs.begin(); k != graphs.end(); ++k) if (k->second.used < old->second.used) old = k;
        graphs.erase(old);
      }
      it = graphs.emplace(key, GraphEntry{}).first;
    }
    GraphEntry& g = it->second;
    if (g.exec && g.gen != ws_gen) { g.exec.reset(); g.seen = 0; }
    g.used = ++graph_clock;
    if (g.exec) {
      CK(cudaGraphLaunch(g.exec, stream));
      ++graph_replays;
      launches += g.nlaunch;
      last_graphed = true;
      return;
    }
    const bool first = (g.seen++ == 0);
    if (first) {                                // first sighting: eager (also performs any workspace growth) ...
      enqueue();
      if (!capture_on_first) return;
    }
    const uint64_t gen0 = ws_gen, l0 = launches;      // ... then capture
    Graph graph;
    CK(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
    capturing = true;
    try {
      enqueue();
    } catch (...) {
      capturing = false;
      cudaStreamEndCapture(stream, graph.out());
      throw;
    }
    capturing = false;
    CK(cudaStreamEndCapture(stream, graph.out()));
    cudaError_t e = cudaGraphInstantiate(g.exec.out(), graph, 0);
    if (e != cudaSuccess) throw Err{VTTS_ERR_CUDA, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e)};
    g.gen = gen0;
    g.nlaunch = launches - l0;
    if (first) { launches = l0; return; }       // (the eager run above already did the work)
    CK(cudaGraphLaunch(g.exec, stream));
    ++graph_replays;
    last_graphed = true;
  }
  // Every kernel goes through here: programmatic dependent launch lets the next kernel's prologue overlap this one's tail.
  template <typename... KArgs, typename... Args>
  void klaunch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, Args&&... args) {
    cudaLaunchConfig_t lc;
    memset(&lc, 0, sizeof(lc));
    lc.gridDim = grid; lc.blockDim = block; lc.dynamicSmemBytes = smem; lc.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    lc.attrs = at;
    lc.numAttrs = use_pdl ? 1 : 0;
    CK(cudaLaunchKernelEx(&lc, kern, static_cast<KArgs>(args)...));
  }
  static uint64_t mix(uint64_t h, uint64_t v) { h ^= v + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2); return h; }

  Tensor tensor(const std::string& name) {
    auto it = tensors.find(name);
    if (it == tensors.end()) throw Err{VTTS_ERR_WEIGHTS, "weight blob has no tensor '" + name + "'"};
    looked_up.push_back(name);
    return it->second;
  }
  std::vector<std::string> looked_up;          // tensors the engine bound, in first-use order
  Buf<PrefRange> d_pref;                       // L2 prefetch list for this precision mode
  int n_pref = 0, n_pref_phase1 = 0;
  bool use_prefetch = false;                   // measured: no gain (weights are not the latency bottleneck)
  void build_prefetch_list();
  const float* vec(const std::string& name, size_t n) {
    Tensor t = tensor(name);
    if (t.n != n) {
      std::ostringstream os;
      os << "tensor '" << name << "' has " << t.n << " elements, expected " << n;
      throw Err{VTTS_ERR_WEIGHTS, os.str()};
    }
    return t.p;
  }
  // need_w = false: the conv runs on wgmma from its split-bf16 copy in this precision mode; the fp32 copy is bound only if
  // the blob happens to carry it (weights.pack(precision=...) leaves it out of the one-time weight broadcast)
  ConvW conv(const std::string& name, int Cin, int Cout, int k, bool need_w = true) {
    ConvW c;
    c.Cin = Cin; c.Cout = Cout; c.k = k; c.ldw = (Cout + 3) / 4 * 4;
    if (need_w || tensors.count(name + ".w")) c.w = vec(name + ".w", (size_t)k * Cin * c.ldw);
    c.b = vec(name + ".b", (size_t)c.ldw);
    REQUIRE(Cin % CV_CK == 0, VTTS_ERR_INVALID, "conv input channels must be a multiple of 16");
    return c;
  }
  LnW ln(const std::string& name, int C) { return LnW{vec(name + ".g", C), vec(name + ".b", C)}; }
  EncLayerW enc_layer(const std::string& p, int Hc, int Fc, int ks, int heads, bool need_w = true) {
    EncLayerW L;
    L.heads = heads;
    const int dk = Hc / heads, nrel = 2 * cfg.window_size + 1;
    L.qkv = conv(p + ".qkv", Hc, 3 * Hc, 1, need_w);
    L.o = conv(p + ".o", Hc, Hc, 1, need_w);
    L.relk = vec(p + ".relk", (size_t)nrel * dk);
    L.relv = vec(p + ".relv", (size_t)nrel * dk);
    L.ln1 = ln(p + ".ln1", Hc);
    L.ffn1 = conv(p + ".ffn1", Hc, Fc, ks, need_w);
    L.ffn2 = conv(p + ".ffn2", Fc, Hc, ks, need_w);
    L.ln2 = ln(p + ".ln2", Hc);
    return L;
  }
  DdsW dds(const std::string& p, int C, int k) {
    DdsW d;
    d.sep_w = vec(p + ".sep_w", (size_t)k * C);
    d.sep_b = vec(p + ".sep_b", C);
    d.ln1 = ln(p + ".ln1", C);
    d.pw = conv(p + ".pw", C, C, 1);
    d.ln2 = ln(p + ".ln2", C);
    return d;
  }

  void bind_rel_tc(EncLayerW& L, const std::string& p) {
    if (!tensors.count(p + ".rkh")) return;       // (blob packed without the tables: the FFMA attention is used)
    L.rk_hi = reinterpret_cast<const __nv_bfloat16*>(vec(p + ".rkh", 16 * 128 / 2));
    L.rk_lo = reinterpret_cast<const __nv_bfloat16*>(vec(p + ".rkl", 16 * 128 / 2));
    L.rv_hi = reinterpret_cast<const __nv_bfloat16*>(vec(p + ".rvh", 16 * 128 / 2));
    L.rv_lo = reinterpret_cast<const __nv_bfloat16*>(vec(p + ".rvl", 16 * 128 / 2));
  }
  TcW tcw(const std::string& name, int Cin, int Cout, int k, bool three = false) {
    TcW t;
    const size_t n = (size_t)k * Cout * Cin / 2;
    t.hi = reinterpret_cast<const __nv_bfloat16*>(vec(name + (three ? ".t3h" : ".th"), n));
    t.lo = reinterpret_cast<const __nv_bfloat16*>(vec(name + (three ? ".t3l" : ".tl"), n));
    if (three) t.mid = reinterpret_cast<const __nv_bfloat16*>(vec(name + ".t3m", n));
    REQUIRE(Cin % TC_BK == 0, VTTS_ERR_INVALID, "tensor-core conv needs input channels in multiples of 64");
    return t;
  }
  Buf<__nv_bfloat16> pl_pool_mid[64];
  Planes planes(int slot, long units, int rm, int C, int extra = 0, bool three = false) {
    Planes p;
    const long rows = units * rm + (extra ? (long)B * extra : 0);
    p.C = C; p.rows = rows;
    const size_t n = (size_t)rows * C + 64;
    REQUIRE(slot >= 0 && 2 * slot + 1 < 128, VTTS_ERR_INVALID, "plane slot out of range");
    const size_t cap_hi = pl_pool[2 * slot].cap, cap_lo = pl_pool[2 * slot + 1].cap;
    p.hi = ensure(pl_pool[2 * slot], n);
    p.lo = ensure(pl_pool[2 * slot + 1], n);
    // fresh device memory may hold NaN bit patterns: rows a kernel never writes (beyond an utterance's end inside the last
    // tile) are multiplied by exact zeros in the attention's P V product, so they must at least be finite
    if (pl_pool[2 * slot].cap != cap_hi) CK(cudaMemsetAsync(p.hi, 0, pl_pool[2 * slot].cap * sizeof(__nv_bfloat16), stream));
    if (pl_pool[2 * slot + 1].cap != cap_lo) CK(cudaMemsetAsync(p.lo, 0, pl_pool[2 * slot + 1].cap * sizeof(__nv_bfloat16), stream));
    if (three) {
      const size_t cap_mid = pl_pool_mid[slot].cap;
      p.mid = ensure(pl_pool_mid[slot], n);
      if (pl_pool_mid[slot].cap != cap_mid) CK(cudaMemsetAsync(p.mid, 0, pl_pool_mid[slot].cap * sizeof(__nv_bfloat16), stream));
    }
    if (collecting) {   // rows behind each utterance must read as zero through TMA: zeroed by one zero_tails launch per phase
      REQUIRE(tail.n < ZT_MAXP && C % 8 == 0, VTTS_ERR_INVALID, "too many plane buffers in one phase");
      TailList::E& e = tail.e[tail.n++];
      e.hi = p.hi; e.lo = p.lo; e.mid = p.mid; e.C = C; e.rm = rm; e.extra = extra; e.rows_cap = (int)rows;
    }
    return p;
  }
  CUtensorMap make_map(const void* base, int C, long rows, int box_rows);
  bool attn_tc_ok(const EncLayerW& L, int Hc, const Tuning& t) const;
  bool attn_use_tc(const EncLayerW& L, int Hc, const Rows& r) const;
  bool attn_split_fits(const EncLayerW& L, int Hc, const Rows& r) const;
  void launch_attn_tc(const Planes& qkv, float* ao, Planes* pl, const EncLayerW& L, int Hc, const Rows& r);
  void launch_tc(const std::vector<TcSpec>& ps, int rmul, const Rows& r);
  // plane buffers of the frame-resolution stages: allocated (and their tails zeroed by ONE zero_tails launch) before the
  // first kernel of the phase
  struct FlowPl { Planes ph, pao, ph1, pff, pwx, pacts, pskip, pqkv; } flp;
  struct DecPl { Planes pz, cur; std::vector<Planes> px, nxt; std::vector<std::vector<Planes>> pj, pt; } dcp;
  void alloc_flow_planes();
  void alloc_decoder_planes();
  bool decoder_tc(float* z, bool pz_ready, const Rows& r);
  void flow_tc(float* z, bool emit_pz, const float* cond, int cond_ld, bool forward, const Rows& r);
  void launch_attn(const float* qkv, float* ao, const EncLayerW& L, int Hc, Planes* pl, const Rows& r);
  void bind_weights();
  void bind_flow_decoder();
  void bind_decoder();
  void bind_wn_encoder(const std::string& p, int cin);
  void launch_conv(const std::vector<ConvP>& ps, int rmul, const Rows& r);
  void encoder_layer(const EncLayerW& L, float*& x, float*& xb, float* qkv, float* ao, float* y, float* ffh, int Hc, int Fc,
                     int ks, const float* vec_after, int vec_ld, const float* cadd_after, const Rows& r);
  void dds_stack(const DdsW* d, int C, int k, float*& a, float*& b, const Rows& r,
                 const float* x0 = nullptr, const float* pre_w = nullptr, const float* pre_b = nullptr, const float* cond = nullptr);
  void dds_layer(const DdsW& d, int C, int k, int dil, const float* x, float* y, const Rows& r,
                 const float* x0 = nullptr, const float* pre_w = nullptr, const float* pre_b = nullptr, const float* cond = nullptr);
  void stage_tokens(const int64_t* ids, int t_max, bool phase1, bool eps);
  void stage1(int t_max, const float* noise_dp_host);
  void finish1();
  Planes enc_px;                               // the text encoder's output planes (precision modes 2 / 3), read by prior_stats
  void text_encoder(const float* cond, int cond_ld);
  void prior_stats();
  void phase1(const int64_t* d_ids64, int t_max, const int64_t* d_sid64, const float* noise_dp, bool noise_on_device);
  void phase2(const float* noise_z, int z_ld, bool noise_on_device, bool run_decoder = true);
  // Per-call scalars prm[0..n): the call's scales (the noise scale, or TTS's three), zeros, the seed's 32-bit halves at [4..5]
  static void put_scalars(float* prm, int n, const float* scales, int nscales, uint64_t seed) {
    std::fill(prm, prm + n, 0.f);
    std::copy(scales, scales + nscales, prm);
    const uint32_t half[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
    memcpy(prm + 4, half, sizeof(half));
  }
  // Caller noise rows [B][I][ld] (memory maybe pageable) -> pinned [B][I][maxFrm]: the first cols[b] columns of item b
  void stage_noise(float* pin, const float* noise, int64_t ld, const std::vector<int>& cols) {
    const int I = cfg.inter_channels;
    for (int b = 0; b < B; ++b)
      for (int ch = 0; ch < I; ++ch)
        memcpy(pin + ((size_t)b * I + ch) * maxFrm, noise + ((size_t)b * I + ch) * ld, (size_t)cols[b] * sizeof(float));
  }
  void stage_noise_z(const float* noise_z, int z_ld) {
    Staging& s = stg[STG_NOISE_Z];
    s.begin();
    s.add(d_eps_z, (size_t)B * cfg.inter_channels * maxFrm);
    s.commit();
    stage_noise(s.host(d_eps_z), noise_z, z_ld, std::vector<int>(B, std::min(z_ld, maxFrm)));
  }
  void decode(float* z, const Rows& r, bool planes_ready = false, bool pz_ready = false);
  // The decoder's element-wise launches, shared by both decoders and the unit-test hooks (vtts_debug_mrf_mean / _istft)
  void mrf_mean(const std::vector<float*>& xj, float* X, long total4);
  void mrf_mean_planes(const std::vector<float*>& xj, float* out, const Planes& nxt, int ch, bool last, int rm, const Rows& r);
  void istft_tail(const float* post, int rm, const Rows& r, float* wav);
  bool have_latent = false;
  Buf<int> d_chunk;                              // [len, off, off_end] of the chunk being decoded

  // WN stack (modules.py:148-176) shared by the flow's coupling layers and the posterior encoder: `x` (and, on the tensor
  // cores, its planes px) is updated in place, `skip` receives the summed skip halves (planes pskip from the last layer);
  // layer i adds the cond rows cond + i*2H (row stride cond_ld) before the gate, none when cond is null.
  void wn_ffma(const std::vector<ConvW>& in, const std::vector<ConvW>& rsx, const std::vector<ConvW>& rss, int nl, int fk,
               int dil_rate, float* x, float* acts, float* skip, const float* cond, int cond_ld, const Rows& r);
  void wn_tc(const std::vector<TcW>& t_in, const std::vector<ConvW>& in, const std::vector<TcW>& t_rsx, const std::vector<ConvW>& rsx,
             const std::vector<TcW>& t_rss, const std::vector<ConvW>& rss, int nl, int fk, int dil_rate, float* x, float* skip, const Planes& px,
             const Planes& pacts, const Planes& pskip, const float* cond, int cond_ld, const Rows& r);
  // The flow on the fp32 pipe; forward = models.py:750-753 (layers in order, x1 <- x1 + m), else the reverse of infer.
  void flow_ffma(float* z, const float* cond, int cond_ld, bool forward, const Rows& r);

  // ---- voice conversion (SynthesizerTrn.voice_conversion, models.py:1710-1718)
  bool has_encq = false, q_tc = false;
  static constexpr int Q_LAYERS = 16, Q_KERNEL = 5;        // PosteriorEncoder(spec_channels, I, H, 5, 1, 16, gin) (models.py:1616)
  static constexpr int QV_UNITS = 768;                     // QuickVC's enc_p = PosteriorEncoder(768, I, H, 5, 1, 16) (vc/models.py:825)
  ConvW q_pre, q_proj;
  std::vector<ConvW> q_in, q_rsx, q_rss;
  std::vector<TcW> qt_in, qt_rsx, qt_rss;
  TcW qt_proj;
  const float *q_cond_w = nullptr, *q_cond_b = nullptr, *stft_basis = nullptr, *mel_fb = nullptr;
  int q_R = 0, spec_pad = 0, vc_pad = 0, vc_wld = 0;
  Buf<int> d_vint;                                 // [clip_len B][sid 2B]
  Buf<float> d_vprm, d_vin, d_vlin, d_vfeat, d_vstats, d_vcsrc, d_vnoise, d_vz_dbg, d_vzp_dbg, d_qg;
  // what a call on recordings stages as its input: waveforms, spectrogram (or log-mel) rows, QuickVC's content-unit rows, or
  // nothing (ContentVec writes the unit rows on the device); the last two also stage QuickVC's target voice g
  enum ClipIn { IN_WAV, IN_SPEC, IN_UNITS, IN_NONE };
  void stage_clip_fields(ClipIn in, bool eps);
  float* vc_upload(bool eps);
  float* cond_src(bool tgt);
  float* front_end(bool from_spec);
  void posterior_encode(const float* feat, int feat_ld, const float* noise, const float* qcond, int qld, const Rows& r);
  void posterior_side(bool from_spec, const float* noise, const float* csrc, const Rows& r);
  void convert_enqueue(bool from_spec, bool eps);

  // ---- QuickVC speaker encoder (SpeakerEncoder.embed_utterance, vc/models.py:728-767; spk.cuh)
  ConvW spk_ih[3];                                 // W_ih x + b_ih + b_hh of each layer, a 1x1 conv
  const float *spk_hh[3] = {}, *spk_lin_w = nullptr, *spk_lin_b = nullptr;
  int spk_nseq = 0, spk_rows = 0;
  int spk_clusters[4] = {};                        // co-resident clusters of lstm_rec_kernel<1 / 2 / 4 / 8>
  Buf<int> d_sseq;                                 // [xrow nseq][len nseq][off nseq + 1][last nseq][seq_of_clip B + 1]
  Buf<float> d_sx[3], d_sh[3], d_sg;
  void bind_quickvc();
  void spk_enqueue(bool from_mel, const std::vector<int>& seq, int max_len);

  // ---- QuickVC conversion (SynthesizerTrn.infer, vc/models.py:862-872): enc_p is bound into the q_* members (the same
  //      16-layer k=5 WN as enc_q, which a QuickVC engine does not hold), the flow and the decoder as in a VITS2 engine
  bool has_encp = false;
  void quickvc_enqueue(bool eps, bool from_wav = false);

  // ---- ContentVec (HubertModel of vc/contentvec.py; contentvec.cuh): waveform -> content-unit rows, fp32 FFMA in every mode
  bool has_cv = false;
  const float *cv_w0 = nullptr, *cv_gn_g = nullptr, *cv_gn_b = nullptr, *cv_fp_g = nullptr, *cv_fp_b = nullptr;
  const float *cv_enc_g = nullptr, *cv_enc_b = nullptr, *cv_pos_w = nullptr, *cv_pos_b = nullptr;
  ConvW cv_conv[8], cv_fp;                         // layers 1.. of the feature encoder: k taps of stride s as one 1x1 conv
  TcW cv_tfp;
  std::vector<EncLayerW> cv_enc;                   // relk / relv point at zeros: the attention's relative terms vanish
  int cv_P = 1;                                    // product of the strides after layer 0
  bool cv_tc = false;                              // precision modes >= 1: the transformer's GEMMs and attention on wgmma
  // shape of the current call: maxS the sample bucket, tot0 the layer-0 rows (a multiple of cv_P), MC GroupNorm chunks per
  // clip, maxL the longest clip of every level (from maxS), nint the int table [lens NL][offs NL][woff][sample mean, float bits] x B
  struct CvPlan { int maxS = 0, tot0 = 0, MC = 0, nint = 0; std::vector<int> maxL; std::vector<int> h; } cvp;
  Buf<int> d_cvi;
  Buf<float> d_cvzero, d_cvwav, d_cvps, d_cvpq, d_cvl[2], d_cvx, d_cvx1, d_cvy, d_cvqkv, d_cvao, d_cvff, d_cvu, d_cvdbg;
  void bind_contentvec();
  std::vector<int> cv_stage(const float* wav, const int64_t* lengths, int64_t ld);
  void cv_enqueue(float* out, const int* out_offs, bool fixed = false);
  // The post-LN transformer layers ContentVec and BERT share, and the launches they are made of: work buffers xa (the input
  // rows, whose planes are PX), xb, Y, QKV, AO, FF and, on the tensor cores, the planes of every GEMM operand
  struct PostLnWs { float *xa, *xb, *Y, *QKV, *AO, *FF; Planes PX, PQKV, PAO, PX1, PFF; };
  void post_ln_layers(const std::vector<EncLayerW>& layers, bool on_tc, int H, int Fh, float eps, PostLnWs w, float* out,
                      const int* out_offs, const Rows& r, bool relu = false, const std::function<void(int)>* after_qkv = nullptr,
                      const int* prefix = nullptr);
  void ln_rows(const float* a, const float* y, const LnW& w, float eps, float* out, const int* out_offs, int C, const Planes* pl,
               const Rows& r);
  void gelu_rows(float* y, int C, const Planes* pl, const Rows& r);
  void gemm_rows(const Planes& in, const TcW& w, const ConvW& cw, float* y, const float* res, const Planes* out, const Rows& r);

  // ---- SoVITS (SynthesizerTrn of GPT-SoVITS module/models.py; sovits.cuh): HuBERT rows -> 25 Hz semantic codes.  HuBERT is
  //      the ContentVec above (cv.*); ssl_proj (k = 2, stride 2) is a 1x1 conv over pair rows, the codebook scores a 1x1 conv
  //      (weight 2E, bias -|E|^2), both fp32 FFMA in every mode, then sv_argmax_kernel.
  ConvW sv_proj, sv_score;
  int sv_K = 0;                                    // codebook entries
  // shape of the current call: B clips, pairs_cap the pair rows the buffers hold (a function of the graph key), maxP the
  // launch's pair rows per clip, h the int table [HuBERT row offsets][pair counts][pair offsets] x B.  Clip b's HuBERT rows
  // start at row 2 q_b, q_b = sum over earlier clips of ceil(frames / 2), so its pair rows (2 frames each) start at q_b.
  struct SvPlan { int pairs_cap = 0, maxP = 0; std::vector<int> h, frames; } svp;
  Buf<int> d_svi, d_svcodes;
  Buf<float> d_svfeat, d_svproj, d_svscore;
  void bind_sovits();
  void sv_stage(const std::vector<int>& frames, int pairs_cap, int maxP, const float* feats = nullptr, int64_t feats_ld = 0);
  void sv_enqueue(bool from_wav);

  // ---- BERT (transformers' BertModel as bert-export.py exports it; bert.cuh): word pieces -> the hidden rows of the last
  //      layer that runs, in StableTTS engines whose blob carries bt.*.  Described by the cv_* fields of vtts_config.
  bool has_bert = false, bt_tc = false;
  int bt_vocab = 0, bt_max_pos = 0;                // rows of the word and position tables
  const float *bt_word = nullptr, *bt_pos = nullptr, *bt_type = nullptr;
  LnW bt_ln;
  std::vector<EncLayerW> bt_enc;
  // shape of the current call: maxL the longest sentence's bucket, tot the rows of the packed sentences (bucketed)
  struct BtPlan { int maxL = 0, tot = 0; std::vector<int> len, off; } btp;
  Buf<int> d_bti;                                  // [len B][off B][ids tot]
  Buf<float> d_btzero, d_btx, d_btx1, d_bty, d_btqkv, d_btao, d_btff, d_btout;
  void bind_bert();
  void bt_stage(const int64_t* ids, const int64_t* lengths, int64_t ld);
  void bt_enqueue(float* out);

  // ---- GPT-SoVITS text-to-semantic decoder (Text2SemanticDecoder.infer_panel; t2s.cuh, DESIGN.md 4.s): the text rows'
  //      prefill on post_ln_layers, then one-token decode steps on the t2s_* kernels, graphed T2S_CHUNK steps at a time
  static constexpr int T2S_CHUNK = 16;
  static constexpr int T2S_BERT = 1024;             // bert_proj's input width (t2s_model.py:54)
  int t2s_text_vocab = 0, t2s_vocab = 0, t2s_npos = 0;
  bool t2s_tc = false;
  float t2s_alpha[2] = {1.f, 1.f};                 // ar_text_position.alpha, ar_audio_position.alpha
  const float *t2s_temb = nullptr, *t2s_aemb = nullptr, *t2s_pe = nullptr;
  ConvW t2s_bp, t2s_pred;
  std::vector<EncLayerW> t2s_enc;
  Buf<float> d_t2s_zero, d_t2s_x, d_t2s_x1, d_t2s_y, d_t2s_qkv, d_t2s_ao, d_t2s_ff, d_t2s_pre, d_t2s_bert, d_t2s_bp;
  Buf<float> d_t2s_k, d_t2s_v, d_t2s_dec, d_t2s_part, d_t2s_q, d_t2s_raw;
  Buf<int> d_t2s_i, d_t2s_st, d_t2s_tok;
  Buf<unsigned> d_t2s_seen;
  Buf<T2sPrm> d_t2s_prm;
  Buf<unsigned long long> d_t2s_seed;
  void bind_t2s();

  // ---- StableTTS flow-matching decoder (CFM.forward / solve_euler / Decoder; dit.cuh): fp32 FFMA in modes 0, 1 and 3; in
  //      mode 2 the convs in stp_tc and the attention on the tensor cores (DESIGN.md 4.r)
  ConvW st_cp[3], st_in, st_final;                 // cond_proj's three convs, in_proj over (x | cond), final_proj
  std::vector<ConvW> st_lsc;                       // the long-skip convs over (x | skip)
  // the pipe of each mel-phase stage in precision mode 2 (all false otherwise): a conv runs on conv_tc_kernel when its input
  // and output widths are multiples of TC_BK (st_tc_fits); in_proj (x | cond) and final_proj stay on the FFMA pipe
  struct StPipe { bool on = false, cp[3] = {false, false, false}, qkv = false, o = false, ffn1 = false, ffn2 = false, lsc = false, attn = false; } stp_tc;
  static bool st_tc_fits(int cin, int cout) { return cin % TC_BK == 0 && cout % TC_BK == 0; }
  TcW st_tcp[3];                                   // split-bf16 weights of cond_proj's convs, of the long skips
  std::vector<TcW> st_tlsc;
  // planes of the mel phase's tensor-core operands: mu, cond_proj's two SiLU outputs, the modulated LayerNorm, q | k | v,
  // the attention output, SiLU(ffn1) and the long-skip operands (null where the consumer runs on the FFMA pipe)
  struct StPl { Planes mu, p0, p1, N, QKV, AO, FF, cat[4]; } stpl;
  // debug_flags & 1 in mode 2: copies of what block 0's plane-writing kernels read and wrote at step 0 (vtts_debug_read
  // "tc_*"): Ttot rows of row_bytes each, taken from rows of pitch_bytes (fp32 rows, or bf16 planes two per float)
  struct Tap { Buf<float> buf; size_t n = 0; };
  std::map<std::string, Tap> st_taps;
  void st_tap(const char* name, const void* src, size_t row_bytes, size_t pitch_bytes) {
    const size_t T = (size_t)stp.Ttot;
    Tap& t = st_taps[name];
    t.n = (T * row_bytes + 3) / 4;
    CK(cudaMemcpy2DAsync(ensure(t.buf, t.n), row_bytes, src, pitch_bytes, row_bytes, T, cudaMemcpyDeviceToDevice, stream));
  }
  void st_tap_planes(const char* hi, const char* lo, const Planes& p, int C, int ld) {
    st_tap(hi, p.hi, (size_t)C * 2, (size_t)ld * 2);
    st_tap(lo, p.lo, (size_t)C * 2, (size_t)ld * 2);
  }
  std::vector<EncLayerW> st_blk;                   // qkv / o / ffn1 / ffn2 of each block; relk / relv point at zeros
  const float *st_tw1 = nullptr, *st_tb1 = nullptr, *st_tw2 = nullptr, *st_tb2 = nullptr, *st_fw = nullptr, *st_fb = nullptr;
  const float *st_aw1 = nullptr, *st_ab1 = nullptr, *st_aw2 = nullptr, *st_ab2 = nullptr;
  const float *st_emb = nullptr, *st_fake_spk = nullptr, *st_fake_content = nullptr, *st_mel_mean = nullptr, *st_mel_std = nullptr;
  // shape of the current call: NS sequences (B, or 2B with guidance: the unconditional branches follow the conditional
  // ones), Ttot rows over all of them, the staged inputs' kinds.  text: the call is phase B of vtts_stabletts_synthesise (mu
  // is expanded on the device from the token rows, pause frames are filled; prior: the expanded mel encoder output too)
  struct StPlan { int NS = 0, steps = 0, Ttot = 0; bool guided = false, noise = false, rows = false, text = false, prior = false; } stp;
  static constexpr int ST_PRM = 16 + 2 * VTTS_CFM_MAX_STEPS;     // prm[16], t of every step, dt of every step
  Buf<int> d_sti;                                  // [len NS][off NS][sid NS][extent NS]
  Buf<float> d_stf, d_stmu, d_stnoise, d_stfilm, d_stada, d_strope, d_stxc, d_stp0, d_stp1, d_stcat[4], d_stx, d_stx2, d_sth, d_stn,
      d_stqkv, d_stao, d_sty, d_stff, d_stv, d_stmel, d_stzero, d_stdbg_n, d_stdbg_qkv;
  void bind_stabletts();
  void st_enqueue();
  // One DiTConVBlock over a ragged batch (diffusion_transformer.py:98-116), shared by the decoder's blocks and the text
  // encoder's: the conditioning and the work buffers of the caller, over the rows r
  struct StBlk {
    int H, F, heads, rd, ald;                      // widths, rotary features, pitch of a sequence's adaLN rows
    const float2* rope;
    const float* ada;                              // [sequences][ald]
    float *Hb, *N, *QKV, *AO, *Y, *FF;
  };
  void st_block(const StBlk& k, const EncLayerW& L, int l, const float* film, const float* xin, int ldi, float* xout, int ldo, bool tap,
                const Rows& r);
  // the same block in precision mode 2 (stp_tc, stpl); xout_pl: the planes of xout's column block, or null
  void st_block_tc(const StBlk& k, const EncLayerW& L, int l, const float* film, const float* xin, int ldi, float* xout, int ldo,
                   const Planes* xout_pl, bool tap, const Rows& r);

  // ---- StableTTS text encoder and durations (TextEncoder.forward, MatchaTTS.synthesise; stabletts.cuh): blobs of
  // weights.pack_stabletts.  Stack 0 is the mel encoder (conditioned on spk_emb), stack 1 dp_encoder (on dur_spk_emb).
  bool st_text = false, st_prior = false;
  struct StEncW { std::vector<EncLayerW> blk; ConvW proj; const float *aw1, *ab1, *aw2, *ab2, *spk; } st_enc[2];
  const float *st_tok_emb = nullptr, *st_punc_emb = nullptr, *st_bert_w = nullptr, *st_bert_b = nullptr;
  Buf<int> d_stti, d_sttd;                         // [tok len B][tok off B][sid B][ids streams x Ttok]; [dur Ttok][first Ttok][frames B]
  Buf<float> d_sttf, d_stbert, d_sttx, d_stte[2], d_sttada, d_sttrope, d_stmumel, d_stmudp, d_stlogw, d_stpau;
  void stt_enqueue(bool prior);
  // vtts_stabletts_synthesise_pieces_wav: BERT of the staged sentences (bt_stage), then each token's row gathered into d_stbert.
  // d_stg holds the token rows' lengths and offsets and each one's source, BERT's packed row btp.off[b] + bert_rows[b][t].
  Buf<int> d_stg;
  void stt_bert_enqueue();

  // ---- StableTTS vocoder (the HiFi-GAN Generator of matcha/hifigan/models.py; hifigan.cuh), bound into the decoder members
  // (dec.*) when the blob carries it.  In precision modes >= 1 the first voc_nt upsampling stages and their MRFs run on the
  // tensor cores, the upsampling conv after them too; conv_pre, the later MRFs and conv_post stay on the FFMA pipe.
  bool has_voc = false;
  int voc_nt = 0;
  Buf<int> d_hgi;                                  // [len B][off B] of vtts_hifigan_vocode
  Buf<float> d_hgmel;                              // the denormalised mel rows the vocoder reads [Tfrm][st_noise]
  void voc_enqueue(const float* mel, const int* fl, const int* fo);

  // ---- resampling of recordings (vtts_resample; resample.cuh): the taps of each rate pair, uploaded on first use
  struct RsTaps { Buf<float> taps; int up = 0, down = 0, K = 0; };
  std::map<std::pair<int, int>, RsTaps> rs_taps;
  Buf<int> d_rsi;                                  // [in_off B][in_len B][out_off B][out_len B][e_off B]
  Buf<float> d_rsin, d_rsout;
  Buf<double> d_rse;                               // frame energies of the trim
  const RsTaps& resample_taps(int up, int down);

  // ---- forced alignment (the alignment of SynthesizerTrn.forward, models.py:1632-1660)
  Buf<float> d_ncent, d_ncent_dbg, d_ascore;       // neg_cent [B][maxFrm][maxTok] (MAS accumulates in place), scores [B]
  Buf<int> d_adur, d_atof;                         // durations (token rows), token of every frame (frame rows)
  void align_enqueue(bool from_spec, bool eps);
};

namespace {

ConvP mk(const ConvW& W, const float* x, int ldx, int xoff, float* y, int ldy, int yoff, int dil, int pad) {
  ConvP p;
  memset(&p, 0, sizeof(p));
  p.x = x; p.w = W.w; p.bias = W.b; p.y = y;
  p.ldx = ldx; p.xoff = xoff; p.ldw = W.ldw; p.ldy = ldy; p.yoff = yoff;
  p.Cin = W.Cin; p.Cout = W.Cout; p.k = W.k; p.dil = dil; p.pad = pad;
  p.out_mul = 1; p.alpha = 1.f; p.pro = PRO_NONE;
  return p;
}

}  // namespace

// Which bound tensors does a call actually read in this precision mode?  (fp32 `.w` copies of convs that run on
// wgmma are skipped, and so are the bf16 `.th/.tl` copies of convs that stay on the FFMA pipe.)
void vtts_engine::build_prefetch_list() {
  auto on_tc = [&](const std::string& nm) {
    if (nm.rfind("enc.", 0) == 0) return cfg.precision >= 2;
    if (nm.rfind("flow.", 0) == 0 || nm.rfind("dec.", 0) == 0) return cfg.precision >= 1;
    return false;
  };
  std::vector<PrefRange> p1, p2;
  std::unordered_map<std::string, bool> seen;
  for (const std::string& nm : looked_up) {
    if (seen[nm]) continue;
    seen[nm] = true;
    const bool is_w = nm.size() > 2 && nm.compare(nm.size() - 2, 2, ".w") == 0;
    const bool is_t = nm.size() > 3 && (nm.compare(nm.size() - 3, 3, ".th") == 0 || nm.compare(nm.size() - 3, 3, ".tl") == 0);
    if (is_w && tensors.count(nm.substr(0, nm.size() - 2) + ".th") && on_tc(nm)) continue;
    if (is_t && !on_tc(nm)) continue;
    if (nm == "emb_g") continue;                 // one row is read
    const Tensor& t = tensors[nm];
    PrefRange r{reinterpret_cast<const char*>(t.p), (unsigned long long)t.n * sizeof(float)};
    const bool phase1 = nm.rfind("enc.", 0) == 0 || nm.rfind("dp.", 0) == 0 || nm.rfind("cond.", 0) == 0;
    (phase1 ? p1 : p2).push_back(r);
  }
  n_pref_phase1 = (int)p1.size();
  p1.insert(p1.end(), p2.begin(), p2.end());
  n_pref = (int)p1.size();
  PrefRange* d = ensure(d_pref, p1.size() + 1);
  CK(cudaMemcpyAsync(d, p1.data(), p1.size() * sizeof(PrefRange), cudaMemcpyHostToDevice, stream));
  CK(cudaStreamSynchronize(stream));
}

void vtts_engine::bind_weights() {
  const vtts_config& c = cfg;
  const int H = c.hidden_channels, I = c.inter_channels, G = c.gin_channels, D = c.dp_filter_channels;
  REQUIRE(H % 32 == 0 && H <= 256 && D % 32 == 0 && D <= 256, VTTS_ERR_INVALID, "hidden/dp channels must be multiples of 32, <= 256");
  REQUIRE((H / c.n_heads) % 32 == 0 && H / c.n_heads <= 128, VTTS_ERR_INVALID, "head dim must be 32/64/96/128");
  const int fheads = c.flow_n_heads > 0 ? c.flow_n_heads : 2;      // models.py:355: the flow's pre_transformer always has 2 heads
  REQUIRE(!c.use_transformer_flows || ((H / fheads) % 32 == 0 && H / fheads <= 128 && H % fheads == 0), VTTS_ERR_INVALID,
          "flow head dim must be 32/64/96/128");
  REQUIRE(c.dp_num_bins >= 1 && c.dp_num_bins <= SPL_MAXB, VTTS_ERR_INVALID, "dp_num_bins must be in [1, 16]");
  REQUIRE(c.dp_kernel_size % 2 == 1 && c.flow_kernel_size % 2 == 1, VTTS_ERR_INVALID, "odd kernels expected");
  REQUIRE(c.n_resblock_kernels <= CV_MAXP, VTTS_ERR_INVALID, "at most 4 resblocks per stage");
  has_g = c.n_speakers > 0 && G > 0;
  const int nl = c.flow_wn_layers, nf = c.flow_n_flows;
  if (has_g) {
    emb_g = vec("emb_g", (size_t)c.n_speakers * G);
    int r = 0;
    if (c.spk_cond_encoder) { r_spk = r; r += H; }
    r_dp = r; r += D;
    r_flow = r; r += nf * nl * 2 * H;
    if (c.decoder_type == 1 && tensors.count("cond.w") && tensors["cond.w"].n == (size_t)(r + c.upsample_initial_channel) * G) {
      r_dec = r; r += c.upsample_initial_channel;      // plain Generator: x = conv_pre(z) + cond(g)  (models.py:874-875)
    }
    condR = r;
    cond_w = vec("cond.w", (size_t)condR * G);
    cond_b = vec("cond.b", condR);
  }
  enc_emb = vec("enc.emb", (size_t)c.n_vocab * H);
  enc.clear();
  enc_on_tc = c.precision >= 2 && H % TC_BK == 0 && c.filter_channels % TC_BK == 0;
  enc_three = enc_on_tc && c.precision == 3;     // exact 3-way split: durations as exact as the fp32 FFMA path
  for (int i = 0; i < c.n_layers; ++i) enc.push_back(enc_layer("enc." + std::to_string(i), H, c.filter_channels, c.kernel_size, c.n_heads, !enc_on_tc));
  enc_proj = conv("enc.proj", H, 2 * I, 1, !enc_on_tc);
  if (enc_on_tc) {
    for (int i = 0; i < c.n_layers; ++i) {
      const std::string p = "enc." + std::to_string(i);
      enc[i].t_qkv = tcw(p + ".qkv", H, 3 * H, 1, enc_three);
      enc[i].t_o = tcw(p + ".o", H, H, 1, enc_three);
      enc[i].t_ffn1 = tcw(p + ".ffn1", H, c.filter_channels, c.kernel_size, enc_three);
      enc[i].t_ffn2 = tcw(p + ".ffn2", c.filter_channels, H, c.kernel_size, enc_three);
      if (!enc_three) bind_rel_tc(enc[i], p);      // (mode 3 keeps the encoder's attention on the fp32 pipe)
    }
    tc_encproj = tcw("enc.proj", H, 2 * I, 1, enc_three);
  }
  dp_pre = conv("dp.pre", H, D, 1);
  dp_proj = conv("dp.proj", D, D, 1);
  for (int i = 0; i < 3; ++i) dp_dds[i] = dds("dp.convs." + std::to_string(i), D, c.dp_kernel_size);
  cf.clear();
  for (int n = 2; n <= c.dp_n_flows; ++n) {
    CfW f;
    const std::string p = "dp.cf" + std::to_string(n);
    f.pre_w = vec(p + ".pre_w", D);
    f.pre_b = vec(p + ".pre_b", D);
    for (int i = 0; i < 3; ++i) f.dds[i] = dds(p + ".convs." + std::to_string(i), D, c.dp_kernel_size);
    f.proj = conv(p + ".proj", D, 3 * c.dp_num_bins - 1, 1);
    cf.push_back(f);
  }
  dp_ea = vec("dp.ea", 4);
  bind_flow_decoder();
  // ---- posterior encoder enc_q + front end (only in blobs packed with posterior=True)
  has_encq = tensors.count("encq.pre.b") > 0;
  if (has_encq) {
    REQUIRE(c.spec_channels > 0 && c.filter_length > 0 && c.hop_length > 0 && c.filter_length % ST_TN == 0 &&
                c.filter_length > c.hop_length && (c.filter_length - c.hop_length) % 2 == 0,
            VTTS_ERR_INVALID, "bad spectrogram configuration (filter_length must be a multiple of 64, above hop_length)");
    REQUIRE(c.win_length == c.filter_length, VTTS_ERR_INVALID, "win_length != filter_length is not supported by the spectrogram front end");
    REQUIRE(!c.use_mel_posterior_encoder || mel_smem_bytes(c.filter_length) <= (size_t)MEL_SMEM_MAX, VTTS_ERR_INVALID,
            "filter_length too large for the mel projection (its spectrum rows must fit in shared memory)");
    REQUIRE(c.use_mel_posterior_encoder ? c.spec_channels == c.n_mel_channels : c.spec_channels == c.filter_length / 2 + 1,
            VTTS_ERR_INVALID, "spec_channels does not match the posterior encoder's input (n_mel_channels / filter_length/2+1)");
    spec_pad = (c.spec_channels + CV_CK - 1) / CV_CK * CV_CK;     // enc_q.pre runs on the FFMA conv: input zero-padded to 16 channels
    vc_pad = (c.filter_length - c.hop_length) / 2;
    bind_wn_encoder("encq", spec_pad);
    if (has_g) {
      q_R = Q_LAYERS * 2 * H;
      q_cond_w = vec("encq.cond.w", (size_t)q_R * G);
      q_cond_b = vec("encq.cond.b", q_R);
    }
    stft_basis = vec("vc.stft", (size_t)c.filter_length * c.filter_length);
    mel_fb = c.use_mel_posterior_encoder ? vec("vc.mel", (size_t)c.n_mel_channels * (c.filter_length / 2 + 1)) : nullptr;
  }
}

// A PosteriorEncoder's pre / 16-layer WN / proj (models.py:813-842) from the blob's <p>.* (weights._pack_wn_encoder) into the
// q_* members: enc_q of a VITS2 engine, enc_p of a QuickVC one.
void vtts_engine::bind_wn_encoder(const std::string& p, int cin) {
  const vtts_config& c = cfg;
  const int H = c.hidden_channels, I = c.inter_channels;
  const bool qfw = !(c.precision >= 1 && H % TC_BK == 0);
  q_pre = conv(p + ".pre", cin, H, 1);
  q_in.clear(); q_rsx.clear(); q_rss.clear(); qt_in.clear(); qt_rsx.clear(); qt_rss.clear();
  for (int i = 0; i < Q_LAYERS; ++i) {
    q_in.push_back(conv(p + ".in" + std::to_string(i), H, 2 * H, Q_KERNEL, qfw));
    if (i < Q_LAYERS - 1) q_rsx.push_back(conv(p + ".rsx" + std::to_string(i), H, H, 1, qfw));
    q_rss.push_back(conv(p + ".rss" + std::to_string(i), H, H, 1, qfw));
  }
  q_proj = conv(p + ".proj", H, 2 * I, 1, qfw);
  q_tc = tc && !qfw;
  if (q_tc) {
    for (int i = 0; i < Q_LAYERS; ++i) {
      qt_in.push_back(tcw(p + ".in" + std::to_string(i), H, 2 * H, Q_KERNEL));
      if (i < Q_LAYERS - 1) qt_rsx.push_back(tcw(p + ".rsx" + std::to_string(i), H, H, 1));
      qt_rss.push_back(tcw(p + ".rss" + std::to_string(i), H, H, 1));
    }
    qt_proj = tcw(p + ".proj", H, 2 * I, 1);
  }
}

// The reverse flow and the decoder (weights._pack_flow_decoder): shared by both model families.
void vtts_engine::bind_flow_decoder() {
  const vtts_config& c = cfg;
  const int H = c.hidden_channels, I = c.inter_channels;
  const int nl = c.flow_wn_layers, nf = c.flow_n_flows;
  const int fheads = c.flow_n_heads > 0 ? c.flow_n_heads : 2;
  flow.clear();
  for (int f = 0; f < nf; ++f) {
    FlowW F;
    const std::string p = "flow." + std::to_string(f);
    const bool fw = !(c.precision >= 1 && H % TC_BK == 0);       // fp32 copies needed? (no: the whole flow but its pre conv is on wgmma)
    F.pre = conv(p + ".pre", I / 2, H, 1);
    if (c.use_transformer_flows) F.tr = enc_layer(p + ".tr", H, H, c.flow_kernel_size, fheads, fw);
    for (int i = 0; i < nl; ++i) {
      F.in.push_back(conv(p + ".in" + std::to_string(i), H, 2 * H, c.flow_kernel_size, fw));
      if (i < nl - 1) F.rsx.push_back(conv(p + ".rsx" + std::to_string(i), H, H, 1, fw));
      F.rss.push_back(conv(p + ".rss" + std::to_string(i), H, H, 1, fw));
    }
    F.post = conv(p + ".post", H, I / 2, 1, fw);
    if (c.precision >= 1 && H % TC_BK == 0) {
      const int fk = c.flow_kernel_size;
      if (c.use_transformer_flows) {
        F.t_qkv = tcw(p + ".tr.qkv", H, 3 * H, 1);
        F.t_o = tcw(p + ".tr.o", H, H, 1);
        F.t_ffn1 = tcw(p + ".tr.ffn1", H, H, fk);
        F.t_ffn2 = tcw(p + ".tr.ffn2", H, H, fk);
        bind_rel_tc(F.tr, p + ".tr");
      }
      for (int i = 0; i < nl; ++i) {
        F.t_in.push_back(tcw(p + ".in" + std::to_string(i), H, 2 * H, fk));
        if (i < nl - 1) F.t_rsx.push_back(tcw(p + ".rsx" + std::to_string(i), H, H, 1));
        F.t_rss.push_back(tcw(p + ".rss" + std::to_string(i), H, H, 1));
      }
      F.t_post = tcw(p + ".post", H, I / 2, 1);
    }
    flow.push_back(F);
  }
  bind_decoder();
}

// The decoder (dec.*): the VITS2 / QuickVC decoders behind the flow, or the StableTTS vocoder (has_voc).
void vtts_engine::bind_decoder() {
  const vtts_config& c = cfg;
  const int I = c.inter_channels;
  tc = c.precision >= 1 && c.precision <= 3;
  voc_nt = 0;
  if (has_voc && tc) {
    // the leading stages whose MRF width is a multiple of 64 (TC_BK) go to the tensor cores, and so does the upsampling conv
    // after them, which hands fp32 rows to the first FFMA stage; conv_post always reads fp32 rows
    REQUIRE(c.resblock_type == 1, VTTS_ERR_INVALID, "unsupported vocoder: in precision modes >= 1 the tensor-core stages take ResBlock1 only");
    int w = c.upsample_initial_channel;
    while (voc_nt < c.n_upsamples && (w / 2) % TC_BK == 0) { w /= 2; ++voc_nt; }
    REQUIRE(voc_nt >= 1 && voc_nt < c.n_upsamples, VTTS_ERR_INVALID,
            "unsupported vocoder for precision modes >= 1: the first stage's width must be a multiple of 64 and the last stage's not "
            "(use precision 0)");
  }
  const bool pre_tc = tc && !has_voc;              // (the vocoder's conv_pre reads 80 mel channels: FFMA)
  dec_pre = conv("dec.pre", I, c.upsample_initial_channel, 7, !pre_tc);
  if (pre_tc) {
    REQUIRE(c.decoder_type == 0 && c.resblock_type == 1, VTTS_ERR_INVALID, "tensor-core mode supports the MB-iSTFT / ResBlock1 decoder");
    tc_pre = tcw("dec.pre", I, c.upsample_initial_channel, 7);
  }
  ups.clear();
  rbs.clear();
  int ch = c.upsample_initial_channel;
  up_total = 1;
  for (int i = 0; i < c.n_upsamples; ++i) {
    const bool up_tc = tc && (!has_voc || i <= voc_nt), mrf_tc = tc && (!has_voc || i < voc_nt);
    // ConvTranspose1d padding: (K-u)/2 in VITS2 (training/vits2/models.py:857-858, 989-990), (K-u+1-i)/2 with output_padding 1-i in
    // QuickVC (vc/models.py:428-430); both make exactly u*T output rows (config.convt_pad checks QuickVC's)
    const int u = c.upsample_rates[i], K = c.upsample_kernel_sizes[i];
    const int p = c.model_family == VTTS_FAMILY_QUICKVC ? (K - u + 1 - i) / 2 : (K - u) / 2;
    UpW U;
    for (int r = 0; r < u; ++r) {
      // polyphase split of ConvTranspose1d (see weights.convt_phases): taps per phase and left padding
      int d_min = -((r + p) / u);
      int d_max = (K - 1 - r - p) / u;
      U.phase.push_back(conv("dec.up" + std::to_string(i) + ".p" + std::to_string(r), ch, ch / 2, d_max - d_min + 1, !up_tc));
      if (up_tc) U.tphase.push_back(tcw("dec.up" + std::to_string(i) + ".p" + std::to_string(r), ch, ch / 2, d_max - d_min + 1));
      U.pad.push_back(d_max);
    }
    ups.push_back(U);
    ch /= 2;
    up_total *= u;
    for (int j = 0; j < c.n_resblock_kernels; ++j) {
      RbW R;
      const std::string p2 = "dec.rb" + std::to_string(i * c.n_resblock_kernels + j);
      for (int d = 0; d < c.n_resblock_dilations; ++d) {
        if (c.resblock_type == 1) {
          R.c1.push_back(conv(p2 + ".c1." + std::to_string(d), ch, ch, c.resblock_kernel_sizes[j], !mrf_tc));
          R.c2.push_back(conv(p2 + ".c2." + std::to_string(d), ch, ch, c.resblock_kernel_sizes[j], !mrf_tc));
          if (mrf_tc) {
            R.t1.push_back(tcw(p2 + ".c1." + std::to_string(d), ch, ch, c.resblock_kernel_sizes[j]));
            R.t2.push_back(tcw(p2 + ".c2." + std::to_string(d), ch, ch, c.resblock_kernel_sizes[j]));
          }
        } else {
          R.c1.push_back(conv(p2 + ".c." + std::to_string(d), ch, ch, c.resblock_kernel_sizes[j]));
        }
        REQUIRE(CV_TT + (c.resblock_kernel_sizes[j] - 1) * c.resblock_dilations[j][d] <= 32 * CV_XR, VTTS_ERR_INVALID,
                "resblock receptive field too wide for the conv tile");
      }
      rbs.push_back(R);
    }
  }
  if (c.decoder_type == 0) {
    const int cps = c.istft_n_fft + 2;
    dec_post = conv("dec.post", ch, c.subbands * cps, 7, !tc);
    if (tc) tc_post = tcw("dec.post", ch, c.subbands * cps, 7);
    istft_basis = vec("dec.istft", (size_t)cps * c.istft_n_fft);
    pqmf = vec("dec.pqmf", (size_t)c.subbands * 63);
    hop = up_total * c.istft_hop * c.subbands;
  } else {
    dec_post = conv("dec.post", ch, 1, 7);
    hop = up_total;
  }
}

// The vocoder of a StableTTS engine over mel rows [rows][st_noise] (utterance b: fl[b] rows from fo[b]) -> d_wav, sample
// offset fo[b] * hop.  The FFMA convs run in one fixed launch shape (Tuning::fixed_ffma), so that in precision mode 0 an
// utterance's waveform does not depend on what it is batched with.
void vtts_engine::voc_enqueue(const float* mel, const int* fl, const int* fo) {
  Rows r = frm_rows();
  r.lens = fl; r.offs = fo; r.tune = tune.fixed_ffma();
  decode(const_cast<float*>(mel), r);
}

CUtensorMap vtts_engine::make_map(const void* base, int C, long rows, int box_rows) {
  CUtensorMap m;
  cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)C * sizeof(__nv_bfloat16)};
  cuuint32_t box[2] = {(cuuint32_t)TC_BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = encode_tiled(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw Err{VTTS_ERR_CUDA, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")"};
  return m;
}

// Split-K plan of a grouped single-wave tensor-core conv launch: the tile width, the cluster size `split` (1, 2, 4 or 8) and
// a split psplit[p] dividing it per problem; a cluster of problem p covers split / psplit[p] tiles.  Every CTA of the launch
// runs at once, so the launch lasts as long as its longest k-loop, max_p ceil(steps_p / psplit[p]), weighted by what one
// k-step moves into shared memory (48 KB at 64-wide tiles, 64 KB at 128-wide: 3 : 4); the per-CTA prologue and epilogue
// are the same for every CTA and drop out.  Constraints: every cluster with an active tile co-resident (cluster_cap),
// at least min_steps k-steps per split CTA.  Equal costs go to fewer CTAs.  With one problem (or equal k-loops) this is
// the widest co-resident split, and 128-wide tiles exactly when they allow a wider split than 64-wide ones.
struct TcSplitIn {
  int n, nb, gx;                 // problems, utterances, row tiles of the grid
  int bn;                        // 64 / 128 pinned, 0: either
  int max_split, min_steps, n_sm;
  int cluster_cap[2][3];         // co-resident clusters of 2/4/8 CTAs at BN 64 / 128
  int steps[TC_MAXP], cout[TC_MAXP], in_extra[TC_MAXP];
  const int* lens;               // [nb] utterance lengths; problem p has lens[b] * rmul + in_extra[p] rows
  int rmul;
  int rt(int p, int b) const { return (lens[b] * rmul + in_extra[p] + TC_BM - 1) / TC_BM; }   // active row tiles
};
struct TcSplitPlan {
  int bn, split, psplit[TC_MAXP];
};
static TcSplitPlan tc_split_plan(const TcSplitIn& in) {
  TcSplitPlan best{in.bn ? in.bn : 64, 1, {1, 1, 1, 1}};
  long best_cost = -1, best_ctas = 0;
  bool wide = true;
  for (int p = 0; p < in.n; ++p) wide = wide && in.cout[p] >= 128;
  for (int wi = 0; wi < 2; ++wi) {
    const int bn = wi ? 128 : 64;
    if (in.bn ? in.bn != bn : (wi && !wide)) continue;
    // clusters[p][l]: clusters of problem p with an active tile when 2^l consecutive tiles share one
    long clusters[TC_MAXP][4] = {};
    long active = 0;
    for (int p = 0; p < in.n; ++p) {
      const int gyp = (in.cout[p] + bn - 1) / bn;
      for (int b = 0; b < in.nb; ++b) clusters[p][0] += (long)in.rt(p, b) * gyp;
      active += clusters[p][0];
    }
    const bool small = active <= in.n_sm;            // (no cluster split fits beside a machine-filling launch)
    for (int p = 0; p < in.n && small; ++p) {
      const int gyp = (in.cout[p] + bn - 1) / bn;
      for (int l = 1; l < 4; ++l) {
        long c = 0, last = -1;
        for (int b = 0; b < in.nb; ++b)
          for (int by = 0; by < gyp; ++by)
            for (int bx = 0, rt = in.rt(p, b); bx < rt; ++bx) {
              const long t = ((long)b * gyp + by) * in.gx + bx;
              if ((t >> l) != last) { ++c; last = t >> l; }
            }
        clusters[p][l] = c;
      }
    }
    for (int ls = 0; (1 << ls) <= std::min(8, in.max_split) && (ls == 0 || small); ++ls) {
      const int sc = 1 << ls;
      // every assignment psplit[p] = 2^e[p] (e <= ls) with at least one problem at the full cluster
      int ncomb = 1;
      for (int p = 0; p < in.n; ++p) ncomb *= ls + 1;
      for (int ci = 0; ci < ncomb; ++ci) {
        long ncl = 0, crit = 0;
        bool full = false, ok = true;
        for (int q = 0, r = ci; q < in.n; ++q, r /= ls + 1) {
          const int e = r % (ls + 1), s = 1 << e;
          ok = ok && (e == 0 || in.steps[q] >= in.min_steps * s);
          full = full || e == ls;
          ncl += clusters[q][ls - e];
          crit = std::max(crit, (long)((in.steps[q] + s - 1) / s));
        }
        if (!ok || !full || (sc > 1 && ncl > in.cluster_cap[wi][ls - 1])) continue;
        const long cost = crit * (wi ? 4 : 3), ctas = ncl * sc;
        if (best_cost < 0 || cost < best_cost || (cost == best_cost && ctas < best_ctas)) {
          best_cost = cost; best_ctas = ctas;
          best.bn = bn; best.split = sc;
          for (int q = 0, r = ci; q < TC_MAXP; ++q, r /= ls + 1) best.psplit[q] = q < in.n ? 1 << (r % (ls + 1)) : 1;
        }
      }
    }
  }
  return best;
}

// Grouped tensor-core conv launch (conv_tc.cuh).  One CTA = 128 rows x 64 output channels of one problem.
void vtts_engine::launch_tc(const std::vector<TcSpec>& ps, int rmul, const Rows& r) {
  const Tuning& t = r.tune;
  const int nB = r.n, maxLen = r.maxLen;
  const std::vector<int>& hl = r.sized;
  // 128-wide channel tiles halve the activation traffic and run the MMA at its smem-operand optimum, but halve the CTA
  // count: used once the launch still fills the machine (batched calls), or when forced (VTTS_TC_BN).
  int BN = 64;
  {
    long ctas128 = 0;
    bool wide = true;
    for (const TcSpec& q : ps) {
      if (q.Cout < 128) wide = false;
      for (int b = 0; b < nB; ++b) ctas128 += (long)((hl[b] * rmul + q.in_extra + TC_BM - 1) / TC_BM) * ((q.Cout + 127) / 128);
    }
    if (wide && ctas128 >= 2 * n_sm) BN = 128;
    if (t.tc_bn == 64 || t.tc_bn == 128) BN = t.tc_bn;
  }
  REQUIRE(!ps.empty() && (int)ps.size() <= TC_MAXP, VTTS_ERR_INVALID, "bad grouped tensor-core conv");
  TcBatch& tb = tc_batch;   // per-engine scratch (2.6 KB: kept off the stack frame of every caller)
  memset(&tb, 0, sizeof(tb));
  int maxCout = 0, maxL = 0, maxNR = TC_BM;
  // Cluster split-K for launches whose tiles leave most SMs idle (single utterances): clusters of `split` CTAs, problem
  // p's tiles each reduced over psplit[p] of them (tc_split_plan).  Decided before the persistent path: a group with more
  // 64-wide tiles than SMs may still fit one wave of split-K clusters at 128-wide tiles (the decoder's second MRF stage:
  // 144 tiles at BN 64, 72 at BN 128).
  int split = 1;
  int psplit[TC_MAXP] = {1, 1, 1, 1};
  int gx = 0;                                // row tiles of the grid
  for (const TcSpec& q : ps) gx = std::max(gx, (maxLen * rmul + q.in_extra + TC_BM - 1) / TC_BM);
  if (t.tc_tall <= 0 && t.tc_split != 1 && (t.tc_bn == 64 || t.tc_bn == 128 || BN == 64)) {
    TcSplitIn in;
    in.n = (int)ps.size(); in.nb = nB; in.gx = gx;
    in.bn = (t.tc_bn == 64 || t.tc_bn == 128) ? t.tc_bn : 0;
    in.max_split = t.tc_split > 1 ? t.tc_split : 8;
    in.min_steps = t.tc_min_steps;
    in.n_sm = n_sm;
    memcpy(in.cluster_cap, tc_cluster_cap, sizeof(in.cluster_cap));
    in.lens = hl.data(); in.rmul = rmul;
    for (int p = 0; p < in.n; ++p) {
      in.steps[p] = ps[p].Cin / TC_BK * ps[p].k;
      in.cout[p] = ps[p].Cout;
      in.in_extra[p] = ps[p].in_extra;
    }
    const TcSplitPlan pl = tc_split_plan(in);
    BN = pl.bn;
    split = pl.split;
    for (int p = 0; p < in.n; ++p) psplit[p] = pl.psplit[p];
  }
  bool mixed = false;                        // (single-wave image only: split > 1)
  for (size_t p = 0; p < ps.size(); ++p) mixed |= psplit[p] != split;
  if (!mixed) for (int& s : psplit) s = split;
  // "Tall" activation tiles (one TMA box of 128 + (k-1)*dil rows per channel chunk, the taps read it through row-shifted
  // descriptors) cut the L2 -> shared-memory traffic of a k-step from A + W to A/k + W.  On machine-filling launches the
  // mainloop is bound by exactly that traffic (64 KB per k-step and SM at 128-wide tiles against 768 tensor-pipe cycles),
  // so they use it by default (VTTS_TC_TALL: 0 auto, 1 always, -1 never); single-utterance launches prefer split-K.
  bool np3 = false;
  long grid_tiles = 0;
  for (const TcSpec& q : ps) {
    if (q.w.mid && q.in.mid) np3 = true;
    grid_tiles += (long)((maxLen * rmul + q.in_extra + TC_BM - 1) / TC_BM) * ((q.Cout + BN - 1) / BN) * nB;
  }
  const bool big = t.tc_persist == 2 || (t.tc_persist && grid_tiles > (long)t.tc_persist_min * n_sm);   // (2: forced, for tests)
  bool tall = split == 1 && (t.tc_tall > 0 || (t.tc_tall == 0 && big));
  for (const TcSpec& q : ps) {
    const int nr = TC_BM + (q.k - 1) * q.dil;
    if (nr > 192) tall = false;              // shared-memory budget of the activation ring (and TMA box <= 256)
    maxNR = std::max(maxNR, nr);
  }
  if (np3) tall = false;
  if (tall) {
    const int ab = (maxNR * 128 + 1023) / 1024 * 1024;
    const int need = BN == 128 ? tc_smem_bytes<128>(ab, 2, 2, tc_wst<128>()) : tc_smem_bytes<64>(ab, 2, 2, tc_wst<64>());
    if (need > 227 * 1024) tall = false;
  }
  if (!tall) maxNR = TC_BM;
  // TMA multicast of the activation tile across the channel-tile CTAs of a cluster: only when every problem of the
  // launch has the same number of channel tiles (no CTA of a cluster may drop out) and the tile is not "tall"
  int cn = 1;
  if (t.tc_mc && !tall) {
    int ny = -1;
    bool same = true;
    for (const TcSpec& q : ps) {
      const int n = (q.Cout + BN - 1) / BN;
      if (ny < 0) ny = n; else if (n != ny) same = false;
    }
    if (same) cn = (ny % 4 == 0) ? 4 : (ny % 2 == 0 ? 2 : 1);
    if (t.tc_mc == 2 && same && ny % 2 == 0) cn = 2;          // VTTS_TC_MULTICAST=2: pairs only
  }
  if (split > 1) cn = 1;
  int np = 0;
  for (const TcSpec& q : ps) {
    const int n = (q.w.mid && q.in.mid) ? 3 : 2;
    REQUIRE(np == 0 || np == n, VTTS_ERR_INVALID, "grouped tensor-core conv mixes 2- and 3-plane problems");
    np = n;
  }
  if (np == 3) { tall = false; cn = 1; }
  tb.np = np;
  tb.ast = (np == 3 || tall) ? 2 : (BN == 128 ? tc_ast<128>() : tc_ast<64>());
  long tiles_all = 0;                        // the launch's CTAs (one wave or less: the one-tile-per-CTA kernel)
  int ncl = 0;                               // mixed splits: clusters of the grid
  if (mixed) {
    for (size_t p = 0; p < ps.size(); ++p) {
      tb.p[p].cl0 = ncl;
      const int m = split / psplit[p];
      ncl += (int)(((long)gx * ((ps[p].Cout + BN - 1) / BN) * nB + m - 1) / m);
    }
    tiles_all = (long)ncl * split;
  } else {
    int mc = 0;
    for (const TcSpec& q : ps) mc = std::max(mc, q.Cout);
    tiles_all = (long)gx * ((mc + BN - 1) / BN) * nB * (long)ps.size() * split;
  }
  const bool one_wave = tiles_all <= n_sm && !(t.tc_persist == 2 && split == 1 && cn == 1);
  tb.wst = np == 3 ? (BN == 128 ? 2 : 3) : (BN == 128 ? tc_wst<128>() : tc_wst<64>());
  tb.split = split;
  tb.cn = cn;
  tb.tall = tall ? 1 : 0;
  // persistent launches: CTA pairs share every weight tile through TMA multicast (conv_tc.cuh)
  const int wmc = (big && t.tc_wmc && split == 1 && cn == 1 && np == 2 && n_sm % 2 == 0) ? 2 : 1;
  tb.baseoff = t.tc_baseoff;
  tb.dbgskip = t.tc_dbgskip;
  tb.a_bytes = (maxNR * 128 + 1023) / 1024 * 1024;
  for (size_t i = 0; i < ps.size(); ++i) {
    const TcSpec& q = ps[i];
    TcProblem& P = tb.p[i];
    const int box_rows = tall ? TC_BM + (q.k - 1) * q.dil : TC_BM / cn;
    P.a_hi = make_map(q.in.hi, q.in.C, q.in.rows, box_rows);
    P.a_lo = make_map(q.in.lo, q.in.C, q.in.rows, box_rows);
    P.w_hi = make_map(q.w.hi, q.Cin, (long)q.k * q.Cout, BN / wmc);
    P.w_lo = make_map(q.w.lo, q.Cin, (long)q.k * q.Cout, BN / wmc);
    if (np == 3) {
      P.a_mid = make_map(q.in.mid, q.in.C, q.in.rows, box_rows);
      P.w_mid = make_map(q.w.mid, q.Cin, (long)q.k * q.Cout, BN);
    }
    P.p_mid = q.out.mid;
    P.bias = q.bias;
    P.res = q.res; P.ldr = q.ldr; P.roff = q.roff;
    P.y = q.y; P.ldy = q.ldy; P.yoff = q.yoff;
    P.cond = q.cond; P.cond_ld = q.cond_ld; P.epi = q.epi;
    P.p_hi = q.out.hi; P.p_lo = q.out.lo; P.ldp = q.out.C; P.poff = q.poff;
    P.Cin = q.Cin; P.Cout = q.Cout; P.k = q.k; P.dil = q.dil; P.pad = q.pad;
    P.out_mul = q.out_mul; P.out_add = q.out_add; P.in_extra = q.in_extra; P.out_seq_extra = q.out_seq_extra;
    P.alpha = q.alpha; P.pl_slope = q.pl_slope;
    P.split = psplit[i];
    REQUIRE(q.in.C == q.Cin, VTTS_ERR_INVALID, "plane width must equal the conv input channels");
    maxCout = std::max(maxCout, q.Cout);
    maxL = std::max(maxL, maxLen * rmul + q.in_extra);
  }
  tb.n = (int)ps.size();
  tb.rmul = rmul;
  tb.dbg = tc_dbg;
  tb.nb = nB;
  dim3 grid((maxL + TC_BM - 1) / TC_BM, (maxCout + BN - 1) / BN, nB * tb.n * split);
  if (grid.x == 0) return;
  tb.wpre = one_wave ? 1 : 0;
  // machine-filling launches: one resident CTA per SM walks the tile space (conv_tc.cuh)
  tb.gx = (int)grid.x; tb.gy = (int)grid.y; tb.gz = (int)grid.z;
  tb.mixed = mixed ? 1 : 0;
  if (mixed) grid = dim3(1, 1, (unsigned)tiles_all);
  tb.persist = 0;
  tb.wmc = 1;
  if (split == 1 && cn == 1 && !tb.wpre && (t.tc_persist == 2 || (t.tc_persist && (long)grid.x * grid.y * grid.z > (long)t.tc_persist_min * n_sm))) {
    tb.persist = 1;
    tb.wmc = wmc;
    grid = dim3((unsigned)n_sm, 1, 1);
  }
  REQUIRE(tb.persist || wmc == 1, VTTS_ERR_INVALID, "tensor-core conv: weight multicast planned for a launch that is not persistent");
  const bool single_wave_image = split > 1 || tb.wpre;
  const bool dyn_image = tb.np != 2 || tb.ast != (BN == 128 ? tc_ast<128>() : tc_ast<64>()) || tb.wst != (BN == 128 ? tc_wst<128>() : tc_wst<64>());
  {
    vtts_conv_report rep{};
    rep.use_tc = 1; rep.bn = BN; rep.split = split; rep.tall = tb.tall; rep.cn = cn; rep.wmc = tb.wmc; rep.persist = tb.persist; rep.np = tb.np;
    rep.ast = tb.ast; rep.wst = tb.wst; rep.image = single_wave_image ? (dyn_image ? 1 : 0) : 2;
    rep.grid_x = (int)grid.x; rep.grid_y = (int)grid.y; rep.grid_z = (int)grid.z;
    for (size_t p = 0; p < ps.size(); ++p) rep.psplit[p] = psplit[p];
    note_conv(rep);
  }
  if (profiling) {
    if (tc_prof_used + 2 > tc_prof_ev.size()) {
      tc_prof_ev.resize(tc_prof_used + 2);
      CK(cudaEventCreate(tc_prof_ev[tc_prof_used].out()));
      CK(cudaEventCreate(tc_prof_ev[tc_prof_used + 1].out()));
    }
    for (const TcSpec& q : ps)
      for (int b = 0; b < nB; ++b)
        tc_prof_flops += 2.0 * ((double)r.real[b] * rmul + q.in_extra) * q.Cout * q.Cin * q.k;   // (true lengths)
    ++tc_prof_launches;
    CK(cudaEventRecord(tc_prof_ev[tc_prof_used], stream));
  }
  {
    cudaLaunchConfig_t lc;
    memset(&lc, 0, sizeof(lc));
    lc.gridDim = grid; lc.blockDim = dim3(TC_THREADS); lc.stream = stream;
    lc.dynamicSmemBytes = BN == 128 ? tc_smem_bytes<128>(tb.a_bytes, tb.np, tb.ast, tb.wst) : tc_smem_bytes<64>(tb.a_bytes, tb.np, tb.ast, tb.wst);
    REQUIRE(lc.dynamicSmemBytes <= 227 * 1024, VTTS_ERR_INVALID, "tensor-core conv: shared-memory budget exceeded");
    cudaLaunchAttribute at[2];
    int na = 0;
    if (cn > 1 || split > 1 || tb.wmc > 1) {
      at[na].id = cudaLaunchAttributeClusterDimension;
      at[na].val.clusterDim.x = tb.wmc; at[na].val.clusterDim.y = cn; at[na].val.clusterDim.z = split;
      ++na;
    }
    if (use_pdl) {
      at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      at[na].val.programmaticStreamSerializationAllowed = 1;
      ++na;
    }
    lc.attrs = at; lc.numAttrs = na;
    // single-wave launches all use the split-capable instantiation (also with split == 1): alternating between two kernel
    // images costs instruction-cache misses on every launch of a latency-bound chain
    if (single_wave_image) {
      if (dyn_image) {
        if (BN == 128) CK(cudaLaunchKernelEx(&lc, conv_tc_kernel<128, true>, tb, r.lens, r.offs));
        else CK(cudaLaunchKernelEx(&lc, conv_tc_kernel<64, true>, tb, r.lens, r.offs));
      } else {                    // the default launches carry the descriptor without the third-plane tensor maps
        // (a one-slot descriptor for the single-conv launches was tried as well: alternating between two kernel images on the
        //  chain cost more than the 2 KB of parameters saved -- conv_tc 723 -> 765 us in-graph)
        const auto tl = tc_lite<TC_MAXP>(tb);
        if (BN == 128) CK(cudaLaunchKernelEx(&lc, conv_tc_kernel<128, false, TC_MAXP>, tl, r.lens, r.offs));
        else CK(cudaLaunchKernelEx(&lc, conv_tc_kernel<64, false, TC_MAXP>, tl, r.lens, r.offs));
      }
    } else {                      // more than one wave of tiles: the persistent kernel (also runs them one per CTA when tb.persist == 0)
      if (BN == 128) CK(cudaLaunchKernelEx(&lc, conv_tc_persist_kernel<128>, tb, r.lens, r.offs));
      else CK(cudaLaunchKernelEx(&lc, conv_tc_persist_kernel<64>, tb, r.lens, r.offs));
    }
  }
  CK(cudaGetLastError());
  if (profiling) {
    CK(cudaEventRecord(tc_prof_ev[tc_prof_used + 1], stream));
    tc_prof_used += 2;
  }
  ++launches;
}

// Attention on the tensor cores (attn_tc.cuh): q, k, v come as the split-bf16 planes the qkv conv's epilogue wrote.
bool vtts_engine::attn_tc_ok(const EncLayerW& L, int Hc, const Tuning& t) const {
  const int dk = Hc / L.heads;
  return t.attn_tc_mode > 0 && L.rk_hi != nullptr && dk % 32 == 0 && dk <= 128 && 2 * cfg.window_size + 1 <= ATC_RS && (3 * Hc) % 8 == 0;
}
// Which attention kernel for this launch?  The tensor-core kernel wins as soon as the launch is throughput bound (batches,
// long utterances: 8.8x at 4765 frames, 2.8x on the flow of a 64-utterance batch).  A single short utterance is latency
// bound -- a 128-row wgmma tile walks its 2-4 key tiles serially while the split-KV FFMA kernel spreads 4 query rows x 4
// key segments over 16 warps of ~80 CTAs -- and keeps the FFMA kernel (measured at 162 frames: 6 vs 19 us per launch in the
// graph).  VTTS_ATTN_TC = 0 never / 1 this rule / 2 always.
bool vtts_engine::attn_use_tc(const EncLayerW& L, int Hc, const Rows& r) const {
  const Tuning& t = r.tune;
  if (!attn_tc_ok(L, Hc, t)) return false;
  if (t.attn_tc_mode >= 2) return true;
  return !((t.attn_rows == 0 || t.attn_rows == 1) && attn_split_fits(L, Hc, r));
}

// Can the split-KV FFMA kernel take this launch?  All key tiles of the longest utterance must be resident in shared memory
// (at most ATS_MAXT tiles, and at most ATS_SMEM_MAX bytes: dk 128 at W 4 overflows from 7 tiles, i.e. 193 positions), and
// the CTAs must fit one wave.
bool vtts_engine::attn_split_fits(const EncLayerW& L, int Hc, const Rows& r) const {
  const int dk = Hc / L.heads, nrel = 2 * cfg.window_size + 1;
  long ctas = 0;
  for (int b = 0; b < r.n; ++b) ctas += (long)((r.sized[b] + ATS_ROWS - 1) / ATS_ROWS) * L.heads;
  const int mt = (r.maxLen + AT_KT - 1) / AT_KT;
  return r.tune.attn_split && mt <= ATS_MAXT && ctas <= n_sm && dk % 32 == 0 && dk <= 128 &&
         (long)attn_split_smem_floats(dk, nrel, mt) * (long)sizeof(float) <= ATS_SMEM_MAX;
}

void vtts_engine::launch_attn_tc(const Planes& qkv, float* ao, Planes* pl, const EncLayerW& L, int Hc, const Rows& r) {
  const int dk = Hc / L.heads;
  AttnTcParams ap;
  memset(&ap, 0, sizeof(ap));
  REQUIRE(qkv.C == 3 * Hc, VTTS_ERR_INVALID, "qkv planes must hold 3*H channels");
  ap.q_hi = make_map(qkv.hi, qkv.C, qkv.rows, ATC_BM);
  ap.q_lo = make_map(qkv.lo, qkv.C, qkv.rows, ATC_BM);
  ap.kv_hi = make_map(qkv.hi, qkv.C, qkv.rows, ATC_KT);
  ap.kv_lo = make_map(qkv.lo, qkv.C, qkv.rows, ATC_KT);
  ap.rk_hi = make_map(L.rk_hi, 128, ATC_RELP, ATC_RELP);
  ap.rk_lo = make_map(L.rk_lo, 128, ATC_RELP, ATC_RELP);
  ap.rv_hi = make_map(L.rv_hi, 128, ATC_RELP, ATC_RELP);
  ap.rv_lo = make_map(L.rv_lo, 128, ATC_RELP, ATC_RELP);
  ap.out = ao; ap.ldo = Hc;
  ap.p_hi = pl ? pl->hi : nullptr; ap.p_lo = pl ? pl->lo : nullptr; ap.ldp = pl ? pl->C : 0;
  ap.n_heads = L.heads; ap.window = cfg.window_size;
  ap.koff = Hc; ap.voff = 2 * Hc;
  dim3 grid((r.maxLen + ATC_BM - 1) / ATC_BM, L.heads, r.n);
  if (grid.x == 0) return;
  last_attn = vtts_attn_report{VTTS_ATTN_TC, dk, 0, (int)grid.x, (int)grid.y, (int)grid.z, atc_smem_bytes(dk)};
  switch (dk / 32) {
    case 1: klaunch(attn_tc_kernel<32>, grid, dim3(ATC_THREADS), (size_t)atc_smem_bytes(32), ap, r.lens, r.offs); break;
    case 2: klaunch(attn_tc_kernel<64>, grid, dim3(ATC_THREADS), (size_t)atc_smem_bytes(64), ap, r.lens, r.offs); break;
    case 3: klaunch(attn_tc_kernel<96>, grid, dim3(ATC_THREADS), (size_t)atc_smem_bytes(96), ap, r.lens, r.offs); break;
    default: klaunch(attn_tc_kernel<128>, grid, dim3(ATC_THREADS), (size_t)atc_smem_bytes(128), ap, r.lens, r.offs); break;
  }
  CK(cudaGetLastError());
  ++launches;
}

void vtts_engine::launch_attn(const float* qkv, float* ao, const EncLayerW& L, int Hc, Planes* pl, const Rows& r) {
  const int maxLen = r.maxLen, rows_per_warp = r.tune.attn_rows;
  const int n_heads = L.heads;
  const int dk = Hc / n_heads, nrel = 2 * cfg.window_size + 1;
  __nv_bfloat16* ph = pl ? pl->hi : nullptr;
  __nv_bfloat16* plo = pl ? pl->lo : nullptr;
  __nv_bfloat16* pmi = pl ? pl->mid : nullptr;
  // register-blocked variant (4 query rows per warp) once the launch is throughput bound
  long rows = 0;
  for (int b = 0; b < r.n; ++b) rows += r.sized[b];
  const int R = (rows_per_warp == 1 || rows_per_warp == 4) ? rows_per_warp : (rows * n_heads >= 8L * 2 * n_sm * 4 ? 4 : 1);
  // single short utterances: split-KV variant (all K/V tiles resident, 4 warps per query row) when it fits one wave
  {
    const int mt = (maxLen + AT_KT - 1) / AT_KT;
    if (R == 1 && attn_split_fits(L, Hc, r)) {
      dim3 grid((maxLen + ATS_ROWS - 1) / ATS_ROWS, n_heads, r.n);
      const size_t smem = (size_t)attn_split_smem_floats(dk, nrel, mt) * sizeof(float);
      last_attn = vtts_attn_report{VTTS_ATTN_SPLIT, dk, 1, (int)grid.x, (int)grid.y, (int)grid.z, (int)smem};
#define ATTN_SPLIT(D) klaunch(attn_split_kernel<D>, grid, dim3(ATS_THREADS), smem, qkv, 3 * Hc, ao, Hc, L.relk, L.relv, n_heads, cfg.window_size, mt, r.lens, r.offs, ph, plo, pmi)
      switch (dk / 32) { case 1: ATTN_SPLIT(1); break; case 2: ATTN_SPLIT(2); break; case 3: ATTN_SPLIT(3); break; default: ATTN_SPLIT(4); break; }
#undef ATTN_SPLIT
      CK(cudaGetLastError());
      ++launches;
      return;
    }
  }
  const int QT = 8 * R;
  dim3 grid((maxLen + QT - 1) / QT, n_heads, r.n);
  const size_t smem = (size_t)attn_smem_floats(dk, nrel, R) * sizeof(float);
  last_attn = vtts_attn_report{R == 4 ? VTTS_ATTN_R4 : VTTS_ATTN_R1, dk, R, (int)grid.x, (int)grid.y, (int)grid.z, (int)smem};
#define ATTN_CASE(D, RR) klaunch(attn_kernel<D, RR>, grid, dim3(AT_THREADS), smem, qkv, 3 * Hc, ao, Hc, L.relk, L.relv, n_heads, cfg.window_size, r.lens, r.offs, ph, plo, pmi)
  if (R == 4) {
    switch (dk / 32) { case 1: ATTN_CASE(1, 4); break; case 2: ATTN_CASE(2, 4); break; case 3: ATTN_CASE(3, 4); break; default: ATTN_CASE(4, 4); break; }
  } else {
    switch (dk / 32) { case 1: ATTN_CASE(1, 1); break; case 2: ATTN_CASE(2, 1); break; case 3: ATTN_CASE(3, 1); break; default: ATTN_CASE(4, 1); break; }
  }
#undef ATTN_CASE
  CK(cudaGetLastError());
  ++launches;
}

// Flow (reverse, models.py:750-757) with every dense conv on the tensor cores.  Producers emit the split-bf16
// planes their consumer needs: FFMA pre-conv, attention and LayerNorm kernels through an extra epilogue output,
// tensor-core convs through theirs.  The Flip folding is the same as in the fp32 path.
void vtts_engine::alloc_flow_planes() {
  const int H = cfg.hidden_channels;
  const long F = Tfrm;
  int slot = 40;    // plane slots 40.. are the flow's (the decoder uses 0..)
  flp.ph = planes(slot++, F, 1, H); flp.pao = planes(slot++, F, 1, H); flp.ph1 = planes(slot++, F, 1, H);
  flp.pff = planes(slot++, F, 1, H); flp.pwx = planes(slot++, F, 1, H); flp.pacts = planes(slot++, F, 1, H);
  flp.pskip = planes(slot++, F, 1, H);
  flp.pqkv = planes(slot++, F, 1, 3 * H);
}

void vtts_engine::alloc_decoder_planes() {
  const vtts_config& c = cfg;
  const long F = Tfrm;
  const int nk = c.n_resblock_kernels, nst = has_voc ? voc_nt : c.n_upsamples;
  int slot = 0;
  dcp.pz = planes(slot++, F, 1, c.inter_channels);
  dcp.cur = planes(slot++, F, 1, c.upsample_initial_channel);
  dcp.px.resize(c.n_upsamples); dcp.nxt.resize(c.n_upsamples); dcp.pj.resize(c.n_upsamples); dcp.pt.resize(c.n_upsamples);
  int rmp = 1, chp = c.upsample_initial_channel;
  for (int i = 0; i < nst; ++i) {
    rmp *= c.upsample_rates[i];
    chp /= 2;
    dcp.px[i] = planes(slot++, F, rmp, chp);
    dcp.pj[i].resize(nk); dcp.pt[i].resize(nk);
    for (int j = 0; j < nk; ++j) { dcp.pj[i][j] = planes(slot++, F, rmp, chp); dcp.pt[i][j] = planes(slot++, F, rmp, chp); }
    dcp.nxt[i] = planes(slot++, F, rmp, chp, (i + 1 == c.n_upsamples) ? 1 : 0);
  }
}

// emit_pz: the post convs of the last two coupling layers also write the split-bf16 planes of their half of z for the
// decoder's conv_pre (dcp.pz), which saves the separate fp32 -> planes pass
// forward: the flow's forward direction (models.py:750-753, x1 <- x1 + m, layers in order) for voice conversion; the
// Flip folding of the packed weights is valid for it when flow_n_flows is even.  cond: the [B][cond_ld] rows of the stacked
// conditioning matrix of the speaker the flow runs for (null: unconditioned).
void vtts_engine::flow_tc(float* z, bool emit_pz, const float* cond, int cond_ld, bool forward, const Rows& r) {
  const vtts_config& c = cfg;
  const int H = c.hidden_channels, I = c.inter_channels, half = I / 2;
  const long F = Tfrm;
  const int nf = c.flow_n_flows, nl = c.flow_wn_layers, fk = c.flow_kernel_size;
  float* h = ensure(d_h, (size_t)F * H);
  float* h1 = ensure(d_h1, (size_t)F * H);
  float* wx = ensure(d_wx, (size_t)F * H);
  float* skip = ensure(d_skip, (size_t)F * H);
  float* fy = ensure(d_fy, (size_t)F * H);
  float* fqkv = ensure(d_fqkv, (size_t)F * 3 * H);
  float* fao = ensure(d_fao, (size_t)F * H);
  Planes ph = flp.ph, pao = flp.pao, ph1 = flp.ph1, pff = flp.pff, pwx = flp.pwx, pacts = flp.pacts, pskip = flp.pskip, pqkv = flp.pqkv;
  dim3 lg((r.maxLen + 3) / 4, r.n);
  for (int s = 0; s < nf; ++s) {
    const int f = forward ? s : nf - 1 - s;
    const FlowW& W = flow[f];
    const bool flipped = ((nf - f) % 2) == 1;
    const int x0off = flipped ? half : 0, x1off = flipped ? 0 : half;
    {
      ConvP p = mk(W.pre, z, I, x0off, h, H, 0, 1, 0);
      Planes& dst = c.use_transformer_flows ? ph : pwx;
      p.p_hi = dst.hi; p.p_lo = dst.lo; p.ldp = H; p.pl_slope = 1.f;
      launch_conv({p}, 1, r);
    }
    float* wn_x = h;
    if (c.use_transformer_flows) {
      if (attn_use_tc(W.tr, H, r)) {
        // q, k, v leave the qkv conv as split-bf16 planes only; attention runs on wgmma (attn_tc.cuh)
        { TcSpec q; q.in = ph; q.w = W.t_qkv; q.bias = W.tr.qkv.b; q.Cin = H; q.Cout = 3 * H; q.out = pqkv; q.pl_slope = 1.f;
          launch_tc({q}, 1, r); }
        launch_attn_tc(pqkv, nullptr, &pao, W.tr, H, r);
      } else {
        { TcSpec q; q.in = ph; q.w = W.t_qkv; q.bias = W.tr.qkv.b; q.Cin = H; q.Cout = 3 * H; q.y = fqkv; q.ldy = 3 * H;
          launch_tc({q}, 1, r); }
        launch_attn(fqkv, fao, W.tr, H, &pao, r);
      }
      { TcSpec q; q.in = pao; q.w = W.t_o; q.bias = W.tr.o.b; q.Cin = H; q.Cout = H; q.y = fy; q.ldy = H;
        launch_tc({q}, 1, r); }
      klaunch(add_ln_kernel, dim3(lg), dim3(128), (size_t)(0), h, fy, W.tr.ln1.g, W.tr.ln1.b, nullptr, nullptr, 0, h1, r.lens, r.offs, H, ph1.hi, ph1.lo, (__nv_bfloat16*)nullptr);
      CK(cudaGetLastError());
      ++launches;
      { TcSpec q; q.in = ph1; q.w = W.t_ffn1; q.bias = W.tr.ffn1.b; q.Cin = H; q.Cout = H; q.k = fk; q.pad = (fk - 1) / 2;
        q.epi = TCE_RELU; q.out = pff; q.pl_slope = 1.f;
        launch_tc({q}, 1, r); }
      { TcSpec q; q.in = pff; q.w = W.t_ffn2; q.bias = W.tr.ffn2.b; q.Cin = H; q.Cout = H; q.k = fk; q.pad = (fk - 1) / 2;
        q.y = fy; q.ldy = H;
        launch_tc({q}, 1, r); }
      klaunch(add_ln_kernel, dim3(lg), dim3(128), (size_t)(0), h1, fy, W.tr.ln2.g, W.tr.ln2.b, h, nullptr, 0, wx, r.lens, r.offs, H, pwx.hi, pwx.lo, (__nv_bfloat16*)nullptr);
      CK(cudaGetLastError());
      ++launches;
      wn_x = wx;
    }
    wn_tc(W.t_in, W.in, W.t_rsx, W.rsx, W.t_rss, W.rss, nl, fk, c.flow_dilation_rate, wn_x, skip, pwx, pacts, pskip,
          cond ? cond + r_flow + f * nl * 2 * H : nullptr, cond_ld, r);
    { TcSpec q; q.in = pskip; q.w = W.t_post; q.bias = W.post.b; q.Cin = H; q.Cout = half; q.alpha = forward ? 1.f : -1.f;
      q.y = z; q.ldy = I; q.yoff = x1off; q.res = z; q.ldr = I; q.roff = x1off;
      if (emit_pz && f <= 1) { q.out = dcp.pz; q.poff = x1off; q.pl_slope = 1.f; }     // this half of z is final now
      launch_tc({q}, 1, r); }
  }
}

void vtts_engine::wn_tc(const std::vector<TcW>& t_in, const std::vector<ConvW>& in, const std::vector<TcW>& t_rsx,
                        const std::vector<ConvW>& rsx, const std::vector<TcW>& t_rss, const std::vector<ConvW>& rss, int nl, int fk,
                        int dil_rate, float* x, float* skip, const Planes& px, const Planes& pacts, const Planes& pskip, const float* cond,
                        int cond_ld, const Rows& r) {
  const int H = cfg.hidden_channels;
  int dil = 1;
  for (int i = 0; i < nl; ++i) {
    { TcSpec q; q.in = px; q.w = t_in[i]; q.bias = in[i].b; q.Cin = H; q.Cout = 2 * H; q.k = fk; q.dil = dil;
      q.pad = dil * (fk - 1) / 2; q.epi = TCE_GATE; q.out = pacts; q.pl_slope = 1.f;
      if (cond) { q.cond = cond + i * 2 * H; q.cond_ld = cond_ld; }
      launch_tc({q}, 1, r); }
    TcSpec qs; qs.in = pacts; qs.w = t_rss[i]; qs.bias = rss[i].b; qs.Cin = H; qs.Cout = H; qs.y = skip; qs.ldy = H;
    if (i > 0) { qs.res = skip; qs.ldr = H; }
    if (i < nl - 1) {
      TcSpec qx; qx.in = pacts; qx.w = t_rsx[i]; qx.bias = rsx[i].b; qx.Cin = H; qx.Cout = H; qx.y = x; qx.ldy = H;
      qx.res = x; qx.ldr = H; qx.out = px; qx.pl_slope = 1.f;
      launch_tc({qx, qs}, 1, r);
    } else {
      qs.out = pskip; qs.pl_slope = 1.f;
      launch_tc({qs}, 1, r);
    }
    dil *= dil_rate;
  }
}

// Decoder on the tensor cores (models.py:1016-1040): every conv consumes the split-bf16 planes written by its
// producer's epilogue; fp32 copies exist only where a residual or the MRF mean needs them.  The StableTTS vocoder runs only
// its first voc_nt stages here, from an FFMA conv_pre that writes the planes, and then the next upsampling conv into fp32
// rows d_stage[voc_nt]: returns false, and decode() continues on the FFMA pipe from there.
bool vtts_engine::decoder_tc(float* z, bool pz_ready, const Rows& r) {
  const vtts_config& c = cfg;
  const int I = c.inter_channels;
  const long F = Tfrm;
  const int nk = c.n_resblock_kernels, nd = c.n_resblock_dilations, nst = has_voc ? voc_nt : c.n_upsamples;
  Planes pz = dcp.pz, cur = dcp.cur;
  const std::vector<Planes>&st_px = dcp.px, &st_nxt = dcp.nxt;
  const std::vector<std::vector<Planes>>&st_pj = dcp.pj, &st_pt = dcp.pt;
  if (!pz_ready && !has_voc) {
    dim3 g((r.maxLen + EW_ROWS - 1) / EW_ROWS, r.n);
    klaunch(split_planes_kernel, dim3(g), dim3(EW_THREADS), (size_t)(0), z, I, pz.hi, pz.lo, I, I, 1.f, 0, 1, r.lens, r.offs);
    CK(cudaGetLastError());
    ++launches;
  }
  int ch = c.upsample_initial_channel;
  if (has_voc) {         // conv_pre on the FFMA pipe, its output handed over as the planes of lrelu(x, 0.1)
    ConvP p = mk(dec_pre, z, I, 0, ensure(d_d0, (size_t)F * ch), ch, 0, 1, 3);
    p.p_hi = cur.hi; p.p_lo = cur.lo; p.ldp = ch; p.pl_slope = 0.1f;
    launch_conv({p}, 1, r);
  } else {
    TcSpec q;
    q.in = pz; q.w = tc_pre; q.bias = dec_pre.b; q.Cin = I; q.Cout = ch; q.k = 7; q.dil = 1; q.pad = 3;
    q.out = cur; q.pl_slope = 0.1f;
    if (r_dec >= 0) { q.cond = d_condv.p + r_dec; q.cond_ld = condR; }     // x = conv_pre(z) + cond(g) (QuickVC, vc/models.py:465)
    if (debug_flags & 1) { q.y = ensure(d_d0, (size_t)F * ch); q.ldy = ch; }
    launch_tc({q}, 1, r);
  }
  int rm = 1;
  if ((int)d_stage.size() < c.n_upsamples) {
    d_stage.resize(c.n_upsamples);
    d_xj.resize(c.n_upsamples);
    d_tmp.resize(c.n_upsamples);
    for (int i = 0; i < c.n_upsamples; ++i) { d_xj[i].resize(nk); d_tmp[i].resize(nk); }
  }
  float* lastX = nullptr;
  for (int i = 0; i < nst; ++i) {
    const int u = c.upsample_rates[i], ch2 = ch / 2;
    const long rows = F * rm * u;
    float* X = ensure(d_stage[i], (size_t)rows * ch2);
    Planes px = st_px[i];
    for (int r0 = 0; r0 < u; r0 += TC_MAXP) {
      std::vector<TcSpec> ps;
      for (int ph = r0; ph < std::min(u, r0 + TC_MAXP); ++ph) {
        TcSpec q;
        q.in = cur; q.w = ups[i].tphase[ph]; q.bias = ups[i].phase[ph].b; q.Cin = ch; q.Cout = ch2;
        q.k = ups[i].phase[ph].k; q.dil = 1; q.pad = ups[i].pad[ph];
        q.y = X; q.ldy = ch2; q.out = px; q.pl_slope = 0.1f; q.out_mul = u; q.out_add = ph;
        ps.push_back(q);
      }
      launch_tc(ps, rm, r);
    }
    rm *= u;
    ch = ch2;
    std::vector<float*> xj(nk);
    std::vector<Planes> pj(nk), pt(nk);
    for (int j = 0; j < nk; ++j) {
      xj[j] = ensure(d_xj[i][j], (size_t)rows * ch);
      pj[j] = st_pj[i][j];
      pt[j] = st_pt[i][j];
    }
    auto rb_pair = [&](int j, int d, TcSpec& a, TcSpec& b2) {
      const RbW& R = rbs[i * nk + j];
      const int k = c.resblock_kernel_sizes[j], dl = c.resblock_dilations[j][d];
      a.in = (d == 0) ? px : pj[j]; a.w = R.t1[d]; a.bias = R.c1[d].b; a.Cin = ch; a.Cout = ch; a.k = k; a.dil = dl;
      a.pad = dl * (k - 1) / 2; a.out = pt[j]; a.pl_slope = 0.1f;
      b2.in = pt[j]; b2.w = R.t2[d]; b2.bias = R.c2[d].b; b2.Cin = ch; b2.Cout = ch; b2.k = k; b2.dil = 1; b2.pad = (k - 1) / 2;
      b2.res = (d == 0) ? X : xj[j]; b2.ldr = ch; b2.y = xj[j]; b2.ldy = ch;
      if (d + 1 < nd) { b2.out = pj[j]; b2.pl_slope = 0.1f; }
    };
    // The nk resblocks of the MRF (models.py:1030-1036) are independent chains of 2*nd convs.  Grouped launches keep them
    // in lock-step, so every step lasts as long as its largest kernel size.  Experiment (VTTS_MRF_BRANCH=1, off): for
    // single utterances each chain runs on its own stream (fork / join with events, also inside the captured graph) with
    // the split-K width that suits its own k-loop -- correct, but the concurrent cluster launches of three streams
    // contend and the step gets slower (1.74 vs 1.62 ms).
    long group_tiles = 0;
    for (int b = 0; b < r.n; ++b) group_tiles += (long)nk * ((r.sized[b] * rm + TC_BM - 1) / TC_BM) * ((ch + 63) / 64);
    const bool branch = mrf_branch && !profiling && nk > 1 && nk - 1 <= 3 && group_tiles <= n_sm;
    if (branch) {
      auto chain = [&](int j) {
        for (int d = 0; d < nd; ++d) {
          TcSpec a, b2;
          rb_pair(j, d, a, b2);
          launch_tc({a}, rm, r);
          launch_tc({b2}, rm, r);
        }
      };
      CK(cudaEventRecord(ev_fork, stream));
      for (int j = nk - 1; j > 0; --j) {              // largest kernel size first; chain 0 on the main stream
        CK(cudaStreamWaitEvent(side[j - 1], ev_fork, 0));
        // the launch code enqueues on `stream`: swap the two owners for this chain and back on every exit
        struct Swap { Stream &a, &b; ~Swap() { std::swap(a, b); } } back{stream, side[j - 1]};
        std::swap(stream, side[j - 1]);
        chain(j);
        CK(cudaEventRecord(ev_join[j - 1], stream));
      }
      chain(0);
      for (int j = 1; j < nk; ++j) CK(cudaStreamWaitEvent(stream, ev_join[j - 1], 0));
    } else {
      for (int d = 0; d < nd; ++d) {
        std::vector<TcSpec> p1(nk), p2(nk);
        // Launches of more than one wave (long utterances, batches) walk the tiles in problem order: the resblock with the
        // longest k-loop (largest kernel size) goes first, so that the last tiles are short ones.  Single-wave launches give
        // each resblock its own split instead (tc_split_plan), where the order does not matter.
        for (int j = 0; j < nk; ++j) rb_pair(j, d, p1[mrf_heavy_first ? nk - 1 - j : j], p2[mrf_heavy_first ? nk - 1 - j : j]);
        launch_tc(p1, rm, r);
        launch_tc(p2, rm, r);
      }
    }
    const bool last = (i + 1 == c.n_upsamples);
    Planes nxt = st_nxt[i];
    mrf_mean_planes(xj, (debug_flags & 1) ? X : nullptr, nxt, ch, last, rm, r);
    cur = nxt;
    lastX = X;
  }
  (void)lastX;
  if (has_voc) {
    const int u = c.upsample_rates[nst], ch2 = ch / 2;
    float* X = ensure(d_stage[nst], (size_t)F * rm * u * ch2);
    for (int r0 = 0; r0 < u; r0 += TC_MAXP) {
      std::vector<TcSpec> ps;
      for (int ph = r0; ph < std::min(u, r0 + TC_MAXP); ++ph) {
        TcSpec q;
        q.in = cur; q.w = ups[nst].tphase[ph]; q.bias = ups[nst].phase[ph].b; q.Cin = ch; q.Cout = ch2;
        q.k = ups[nst].phase[ph].k; q.dil = 1; q.pad = ups[nst].pad[ph];
        q.y = X; q.ldy = ch2; q.out_mul = u; q.out_add = ph;
        ps.push_back(q);
      }
      launch_tc(ps, rm, r);
    }
    return false;
  }
  const int cps = c.istft_n_fft + 2, pc = c.subbands * cps;
  float* post = ensure(d_post, ((size_t)F * rm + B) * pc);
  {
    TcSpec q;
    q.in = cur; q.w = tc_post; q.bias = dec_post.b; q.Cin = ch; q.Cout = pc; q.k = 7; q.dil = 1; q.pad = 3;
    q.y = post; q.ldy = pc; q.in_extra = 1; q.out_seq_extra = 1;
    launch_tc({q}, rm, r);
  }
  istft_tail(post, rm, r, ensure(d_wav, (size_t)F * hop + 16));
  return true;
}

// MRF mean of the FFMA decoder over whole stage buffers (total4 float4 units: rows outside the utterances too).
void vtts_engine::mrf_mean(const std::vector<float*>& xj, float* X, long total4) {
  const int nk = (int)xj.size();
  REQUIRE(nk <= 3, VTTS_ERR_INVALID, "more than 3 resblocks per stage not supported");
  klaunch(mrf_mean_kernel, dim3((unsigned)((total4 + 255) / 256)), dim3(256), (size_t)(0), xj[0], nk > 1 ? xj[1] : nullptr, nk > 2 ? xj[2] : nullptr,
          std::min(nk, 3), X, total4);
  CK(cudaGetLastError());
  ++launches;
}

// MRF mean of the tensor-core decoder over the utterances' rows -> planes of lrelu(mean) (the last stage: slope 0.01 and the
// ReflectionPad1d((1,0)) row, models.py:1038-1039), and the fp32 mean into `out` when it is not null.
void vtts_engine::mrf_mean_planes(const std::vector<float*>& xj, float* out, const Planes& nxt, int ch, bool last, int rm, const Rows& r) {
  const int nk = (int)xj.size();
  dim3 g((r.maxLen * rm + (last ? 1 : 0) + EW_ROWS - 1) / EW_ROWS, r.n);
  klaunch(mrf_mean_planes_kernel, dim3(g), dim3(EW_THREADS), (size_t)(0), xj[0], nk > 1 ? xj[1] : nullptr, nk > 2 ? xj[2] : nullptr, std::min(nk, 3),
          out, nxt.hi, nxt.lo, ch, last ? 0.01f : 0.1f, last ? 1 : 0, rm, r.lens, r.offs);
  CK(cudaGetLastError());
  ++launches;
}

// iSTFT + synthesis filter (istft_pqmf_kernel) over the conv_post rows `post` (utterance b: frames rm * len + 1 from row
// offs[b] * rm + b) -> packed waveform rows (utterance b from sample offs[b] * hop).
void vtts_engine::istft_tail(const float* post, int rm, const Rows& r, float* wav) {
  const vtts_config& c = cfg;
  const int pc = c.subbands * (c.istft_n_fft + 2);
  const int M = r.maxLen * rm * c.istft_hop;
  dim3 g((M + TL_M - 1) / TL_M, r.n);
  const size_t smem = ((size_t)tl_rec_frames(63, c.subbands, c.istft_n_fft, c.istft_hop) * pc + (size_t)c.subbands * (TL_M + 2 * tl_halo(63, c.subbands))) * sizeof(float);
  REQUIRE(c.istft_hop == 4 && c.istft_n_fft == 16, VTTS_ERR_INVALID, "iSTFT tail kernel is sized for n_fft=16, hop=4");
  klaunch(istft_pqmf_kernel, dim3(g), dim3(TL_THREADS), (size_t)(smem), post, pc, istft_basis, pqmf, c.subbands, c.istft_n_fft, c.istft_hop, 63, rm, r.lens, r.offs, wav, 0, 1, istft_w2);
  CK(cudaGetLastError());
  ++launches;
}

void vtts_engine::launch_conv(const std::vector<ConvP>& ps, int rmul, const Rows& r) {
  const Tuning& t = r.tune;
  const int nB = r.n, maxLen = r.maxLen;
  ConvBatch cb;
  memset(&cb, 0, sizeof(cb));
  REQUIRE(!ps.empty() && (int)ps.size() <= CV_MAXP, VTTS_ERR_INVALID, "bad grouped conv");
  int maxCout = 0, maxHalo = 0, maxL = 0;
  for (size_t i = 0; i < ps.size(); ++i) {
    cb.p[i] = ps[i];
    maxCout = std::max(maxCout, ps[i].Cout);
    maxHalo = std::max(maxHalo, (ps[i].k - 1) * ps[i].dil);
    maxL = std::max(maxL, maxLen * rmul + ps[i].in_extra);
    REQUIRE(CV_TT + (ps[i].k - 1) * ps[i].dil <= 32 * CV_XR, VTTS_ERR_INVALID, "conv tile halo too large");
  }
  cb.n = (int)ps.size();
  cb.rmul = rmul;
  long base0 = 0;
  for (const ConvP& q : ps)
    for (int b = 0; b < nB; ++b) base0 += (long)((r.sized[b] * rmul + q.in_extra + CV_TT - 1) / CV_TT) * ((q.Cout + CV_TC - 1) / CV_TC);
  // many tiles (batched calls): one thread group per CTA (several CTAs per SM; r2, batch 64: 6.98 ms per step against 8.01 / 8.21
  // with 2 / 4 groups), no cluster.  Few tiles (batch 1): the k-steps of a tile are
  // spread over a cluster of S CTAs until the launch fills ~1 wave of SMs; ranks that still have long k-loops then get
  // 2-4 thread groups each (a lone warp per scheduler issues an FFMA only every other cycle).
  int G = base0 >= 2 * n_sm ? t.conv_big_g : t.conv_min_g;
  for (const ConvP& q : ps)
    while (G > 1 && q.Cin % (CV_CK * G) != 0) G >>= 1;
  auto min_steps = [&](int g) {
    int ms = 1 << 30;
    for (const ConvP& q : ps) ms = (q.Cin % (CV_CK * g) != 0) ? 0 : std::min(ms, q.Cin / (CV_CK * g) * q.k);
    return ms;
  };
  int S = 1;
  while (S < t.conv_max_s && base0 * S < t.conv_target && S * 2 <= min_steps(G)) S *= 2;
  const int xw = (CV_TT + maxHalo + 7) / 8 * 8 + 1;
  auto smem_floats = [&](int g) {
    const size_t pipe = (size_t)2 * CV_CK * g * xw + (size_t)CV_NS * CV_CK * g * CV_TC;
    return (std::max(pipe, (size_t)(g - 1) * 32 * CV_THREADS) + 3) / 4 * 4 + (size_t)32 * CV_THREADS;
  };
  if (t.conv_auto_g && base0 < 2 * n_sm)
    while (G * 2 <= t.conv_max_g && min_steps(G * 2) / S >= t.conv_auto_g && smem_floats(G * 2) * sizeof(float) <= (size_t)CONV_SMEM_MAX) G *= 2;
  REQUIRE(smem_floats(G) * sizeof(float) <= (size_t)CONV_SMEM_MAX, VTTS_ERR_INVALID, "conv tile does not fit in shared memory");
  cb.S = S;
  cb.xw = xw;
  const size_t pipe_floats = (size_t)2 * CV_CK * G * xw + (size_t)CV_NS * CV_CK * G * CV_TC;
  const size_t red_floats = (size_t)(G - 1) * 32 * CV_THREADS;
  const size_t stage_off = (std::max(pipe_floats, red_floats) + 3) / 4 * 4;
  cb.stage_off = (int)stage_off;
  const size_t smem = (stage_off + (S > 1 ? (size_t)32 * CV_THREADS : 0)) * sizeof(float);
  dim3 grid(((maxL + CV_TT - 1) / CV_TT) * S, (maxCout + CV_TC - 1) / CV_TC, nB * cb.n);
  if (grid.x == 0) return;
  {
    vtts_conv_report rep{};
    rep.S = S; rep.G = G;
    rep.grid_x = (int)grid.x; rep.grid_y = (int)grid.y; rep.grid_z = (int)grid.z;
    note_conv(rep);
  }
  if (profiling) {
    if (prof_used + 2 > prof_ev.size()) {
      prof_ev.resize(prof_used + 2);
      CK(cudaEventCreate(prof_ev[prof_used].out()));
      CK(cudaEventCreate(prof_ev[prof_used + 1].out()));
    }
    for (const ConvP& q : ps)
      for (int b = 0; b < nB; ++b)
        prof_flops += 2.0 * ((double)r.real[b] * rmul + q.in_extra) * q.Cout * q.Cin * q.k;
    ++prof_launches;
    CK(cudaEventRecord(prof_ev[prof_used], stream));
  }
  {
    cudaLaunchConfig_t lc;
    memset(&lc, 0, sizeof(lc));
    lc.gridDim = grid;
    lc.blockDim = dim3(CV_THREADS * G);
    lc.dynamicSmemBytes = smem;
    lc.stream = stream;
    cudaLaunchAttribute at[2];
    int na = 0;
    if (S > 1) {
      at[na].id = cudaLaunchAttributeClusterDimension;
      at[na].val.clusterDim.x = S;
      at[na].val.clusterDim.y = 1;
      at[na].val.clusterDim.z = 1;
      ++na;
    }
    if (use_pdl) {
      at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      at[na].val.programmaticStreamSerializationAllowed = 1;
      ++na;
    }
    lc.attrs = at;
    lc.numAttrs = na;
    switch (G) {
      case 4: CK(cudaLaunchKernelEx(&lc, conv_kernel<4>, cb, r.lens, r.offs)); break;
      case 2: CK(cudaLaunchKernelEx(&lc, conv_kernel<2>, cb, r.lens, r.offs)); break;
      default: CK(cudaLaunchKernelEx(&lc, conv_kernel<1>, cb, r.lens, r.offs)); break;
    }
  }
  CK(cudaGetLastError());
  if (profiling) {
    CK(cudaEventRecord(prof_ev[prof_used + 1], stream));
    prof_used += 2;
  }
  ++launches;
}

// One relative-attention encoder layer (attentions.py:57-63): x <- LN2(x1 + FFN(x1)), x1 = LN1(x + MHA(x)).
void vtts_engine::encoder_layer(const EncLayerW& L, float*& x, float*& xb, float* qkv, float* ao, float* y, float* ffh, int Hc,
                                int Fc, int ks, const float* vec_after, int vec_ld, const float* cadd_after, const Rows& r) {
  launch_conv({mk(L.qkv, x, Hc, 0, qkv, 3 * Hc, 0, 1, 0)}, 1, r);
  launch_attn(qkv, ao, L, Hc, nullptr, r);
  launch_conv({mk(L.o, ao, Hc, 0, y, Hc, 0, 1, 0)}, 1, r);
  dim3 lg((r.maxLen + 3) / 4, r.n);
  klaunch(add_ln_kernel, dim3(lg), dim3(128), (size_t)(0), x, y, L.ln1.g, L.ln1.b, nullptr, nullptr, 0, xb, r.lens, r.offs, Hc, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr);
  CK(cudaGetLastError());
  ++launches;
  {
    ConvP p = mk(L.ffn1, xb, Hc, 0, ffh, Fc, 0, 1, (ks - 1) / 2);
    p.epi = EPI_RELU;
    launch_conv({p}, 1, r);
  }
  launch_conv({mk(L.ffn2, ffh, Fc, 0, y, Hc, 0, 1, (ks - 1) / 2)}, 1, r);
  klaunch(add_ln_kernel, dim3(lg), dim3(128), (size_t)(0), xb, y, L.ln2.g, L.ln2.b, cadd_after, vec_after, vec_ld, x, r.lens, r.offs, Hc, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr);
  CK(cudaGetLastError());
  ++launches;
}

void vtts_engine::dds_stack(const DdsW* d, int C, int k, float*& a, float*& b, const Rows& r,
                            const float* x0, const float* pre_w, const float* pre_b, const float* cond) {
  int dil = 1;
  for (int i = 0; i < 3; ++i) {
    dds_layer(d[i], C, k, dil, a, b, r, i == 0 ? x0 : nullptr, pre_w, pre_b, cond);
    std::swap(a, b);
    dil *= k;
  }
}

// One DDSConv layer x -> y; with x0 set the layer's input is the ConvFlow front pre_w * x0 + pre_b + cond instead of x.
void vtts_engine::dds_layer(const DdsW& d, int C, int k, int dil, const float* x, float* y, const Rows& r,
                            const float* x0, const float* pre_w, const float* pre_b, const float* cond) {
  DdsP P;
  P.x = x; P.y = y;
  P.x0 = x0; P.pre_w = pre_w; P.pre_b = pre_b; P.cond = cond;
  P.sep_w = d.sep_w; P.sep_b = d.sep_b;
  P.ln1g = d.ln1.g; P.ln1b = d.ln1.b;
  P.pw_w = d.pw.w; P.pw_b = d.pw.b; P.ldw = d.pw.ldw;
  P.ln2g = d.ln2.g; P.ln2b = d.ln2.b;
  P.C = C; P.k = k; P.dil = dil;
  // (16 positions per CTA were tried for batched calls -- 4x less weight streaming per position -- and measured slower:
  //  duration stage 3.20 vs 2.95 ms at batch 64)
  dim3 grid((r.maxLen + DDS_TT - 1) / DDS_TT, r.n);
  const size_t smem = ((size_t)DDS_NS * DDS_CH * C + (size_t)C * DDS_TT + 8 * DDS_TT) * sizeof(float);
  klaunch(dds_layer_kernel<DDS_TT>, dim3(grid), dim3(C), (size_t)(smem), P, r.lens, r.offs);
  CK(cudaGetLastError());
  ++launches;
}

// ---------------------------------------------------------------------------------------------------
// Phase 1: speaker vector, TextEncoder, StochasticDurationPredictor(reverse), durations.
// ---------------------------------------------------------------------------------------------------
void vtts_engine::phase1(const int64_t* d_ids64, int t_max, const int64_t* d_sid64, const float* noise_dp, bool noise_on_device) {
  const vtts_config& c = cfg;
  const int H = c.hidden_channels, D = c.dp_filter_channels;
  const size_t T = (size_t)Ttok;
  if (!capturing) CK(cudaEventRecord(ev[0], stream));
  // ---- inputs (host data was staged by stage_tokens() and stage1(); only device work is enqueued here;
  //      d_ids64 null: the ids and speaker ids were staged by the host too)
  int* tl = ensure(d_tok_len, B);
  int* to = ensure(d_tok_off, B + 1);
  int* ids = ensure(d_ids, T);
  int* sid = ensure(d_sid, B);
  float* prm = ensure(d_prm, 8);
  const Rows r = tok_rows();
  stg[STG_TOKENS].upload();
  if (d_ids64) {
    dim3 g((maxTok + 127) / 128, B);
    klaunch(pack_ids_kernel, dim3(g), dim3(128), (size_t)(0), d_ids64, t_max, ids, tl, to);
    CK(cudaGetLastError());
    klaunch(cast_sid_kernel, dim3((B + 127) / 128), dim3(128), (size_t)(0), d_sid64, sid, B);
    CK(cudaGetLastError());
    launches += 2;
  }
  if (noise_dp && !noise_on_device) noise_dp = d_eps_dp.p;     // staged as [B][2][maxTok] (stage1)
  if (!capturing) CK(cudaEventRecord(ev[1], stream));

  if (use_prefetch && n_pref > 0) {
    // encoder / duration-predictor weights first, then flow + decoder (needed ~1 ms later)
    klaunch(l2_prefetch_kernel, dim3(8, 64), dim3(256), (size_t)0, (const PrefRange*)d_pref.p, n_pref, 0, n_pref_phase1);
    klaunch(l2_prefetch_kernel, dim3(8, 64), dim3(256), (size_t)0, (const PrefRange*)d_pref.p, n_pref, n_pref_phase1, n_pref);
    launches += 2;
  }
  // ---- speaker conditioning (models.py:1680-1683)
  float* condv = nullptr;
  if (has_g) {
    condv = ensure(d_condv, (size_t)B * condR);
    dim3 g((condR + 7) / 8, B);
    klaunch(cond_kernel, dim3(g), dim3(256), (size_t)(c.gin_channels * sizeof(float)), emb_g, sid, cond_w, cond_b, condv, c.gin_channels, condR, c.n_speakers);
    CK(cudaGetLastError());
    ++launches;
  }
  text_encoder(condv, condR);
  float* x = d_x.p;
  // (the prior projection enc_p.proj, models.py:323, is only needed by phase 2: it is enqueued at the end of this phase so
  //  that it runs while the host picks up the utterance lengths)
  if (!capturing) CK(cudaEventRecord(ev[2], stream));

  // ---- stochastic duration predictor, reverse (models.py:56-63, 93-101)
  float* dA = ensure(d_dA, T * D);
  float* dB = ensure(d_dB, T * D);
  float* dx = ensure(d_dx, T * D);
  // spline parameters of a ConvFlow (3 * nbins - 1 per token; rows padded to float4)
  const int nbins = c.dp_num_bins, ldh = spline_pitch(nbins);
  float* spl = ensure(d_spl, T * ldh);
  float* za = ensure(d_za, T);
  float* zb = ensure(d_zb, T);
  {
    ConvP p = mk(dp_pre, x, H, 0, dA, D, 0, 1, 0);
    if (has_g) { p.cond = condv + r_dp; p.cond_ld = condR; }
    launch_conv({p}, 1, r);
  }
  {
    float *a = dA, *b = dB;
    dds_stack(dp_dds, D, c.dp_kernel_size, a, b, r);
    launch_conv({mk(dp_proj, a, D, 0, dx, D, 0, 1, 0)}, 1, r);
  }
  {
    dim3 g((maxTok + 127) / 128, B);
    klaunch(dp_noise_kernel, dim3(g), dim3(128), (size_t)(0), noise_dp, eps_dp_ld, prm, za, zb, tl, to);
    CK(cudaGetLastError());
    ++launches;
  }
  float* cvar = zb;   // conditioning half (x0 after the Flip)
  float* tvar = za;   // transformed half (x1)
  for (int n = c.dp_n_flows; n >= 2; --n) {
    const CfW& F = cf[n - 2];
    // (the ConvFlow front h = pre(x0) + cond, modules.py:366-367, is computed inside the first DDS layer)
    float *a = dA, *b = dB;
    dds_stack(F.dds, D, c.dp_kernel_size, a, b, r, cvar, F.pre_w, F.pre_b, dx);
    launch_conv({mk(F.proj, a, D, 0, spl, ldh, 0, 1, 0)}, 1, r);
    {
      dim3 g((maxTok + 127) / 128, B);
      klaunch(spline_inverse_kernel, dim3(g), dim3(128), (size_t)(0), spl, ldh, tvar, nbins, c.dp_tail_bound, sqrtf((float)D), tl, to);
      CK(cudaGetLastError());
      ++launches;
    }
    std::swap(cvar, tvar);
  }
  // after the last Flip channel 0 is the half transformed last (== cvar after the swap)
  const float* zlast = (c.dp_n_flows >= 2) ? cvar : za;
  int* wceil = ensure(d_wceil, T);
  int* cum = ensure(d_cum, T);
  int* fl = ensure(d_frm_len, B);
  int* fo = ensure(d_frm_off, B + 1);
  unsigned int* dctr = reinterpret_cast<unsigned int*>(ensure(d_done_ctr, 4));
  int* fl_real = ensure(d_frm_len_real, B);
  klaunch(duration_kernel, dim3(B), dim3(256), (size_t)(0), zlast, dp_ea, 0, 2, prm, wceil, cum, fl, tl, to, fo, B,
          (volatile int*)(use_poll ? map.d : nullptr), dctr, fl_real);
  CK(cudaGetLastError());
  ++launches;
  if (!capturing) CK(cudaEventRecord(ev[3], stream));
  if (!use_poll) stg[STG_LENGTHS].download();
  // prior statistics m_p, logs_p (models.py:323-325): overlaps the host's round trip between the two phases
  prior_stats();
}

// TextEncoder up to its projection (models.py:317-322): embedding, the n_layers relative-attention layers in the precision
// mode's variant -> d_x (and, on the tensor cores, its planes enc_px).  cond: [B][cond_ld] conditioning rows of the speaker
// (the spk_emb_linear rows at r_spk are read), null for an unconditioned model.  Token shape and d_tok_len / d_tok_off / d_ids
// must be set.  Used by phase 1 (TTS) and by the alignment.
void vtts_engine::text_encoder(const float* cond, int cond_ld) {
  const vtts_config& c = cfg;
  const int H = c.hidden_channels, Fc = c.filter_channels;
  const size_t T = (size_t)Ttok;
  const int* tl = d_tok_len.p;
  const int* to = d_tok_off.p;
  const int* ids = d_ids.p;
  const Rows r = tok_rows();
  const float* spk_vec = (cond && r_spk >= 0) ? cond + r_spk : nullptr;

  // ---- text encoder (models.py:317-326)
  float* x = ensure(d_x, T * H);
  float* xb = ensure(d_xb, T * H);
  float* qkv = ensure(d_qkv, T * 3 * H);
  float* ao = ensure(d_ao, T * H);
  float* y = ensure(d_y, T * H);
  float* ffh = ensure(d_ffh, T * Fc);
  Planes& px = enc_px;
  Planes px1, pao, pff, pqkv;
  if (enc_on_tc) {
    begin_planes();
    px = planes(60, (long)T, 1, H, 0, enc_three); px1 = planes(61, (long)T, 1, H, 0, enc_three);
    pao = planes(62, (long)T, 1, H, 0, enc_three); pff = planes(63, (long)T, 1, Fc, 0, enc_three);
    pqkv = planes(59, (long)T, 1, 3 * H);
    flush_tails(tl, to);
  }
  {
    dim3 g(maxTok, B);
    klaunch(embed_kernel, dim3(g), dim3(64), (size_t)(0), ids, enc_emb, x, tl, to, H, sqrtf((float)H), c.n_vocab,
            (spk_vec && c.cond_layer_idx == 0) ? spk_vec : (const float*)nullptr, cond_ld, px.hi, px.lo, px.mid);
    CK(cudaGetLastError());
    ++launches;
  }
  for (int i = 0; i < c.n_layers; ++i) {
    const float* va = (spk_vec && c.cond_layer_idx == i + 1) ? spk_vec : nullptr;
    if (!enc_on_tc) {
      encoder_layer(enc[i], x, xb, qkv, ao, y, ffh, H, Fc, c.kernel_size, va, cond_ld, nullptr, r);
      continue;
    }
    // precision mode 2: same layer with the four convs on wgmma (attentions.py:57-63)
    const EncLayerW& L = enc[i];
    const int ks = c.kernel_size;
    dim3 lg((maxTok + 3) / 4, B);
    if (attn_use_tc(L, H, r)) {
      { TcSpec q; q.in = px; q.w = L.t_qkv; q.bias = L.qkv.b; q.Cin = H; q.Cout = 3 * H; q.out = pqkv; q.pl_slope = 1.f;
        launch_tc({q}, 1, r); }
      launch_attn_tc(pqkv, nullptr, &pao, L, H, r);
    } else {
      { TcSpec q; q.in = px; q.w = L.t_qkv; q.bias = L.qkv.b; q.Cin = H; q.Cout = 3 * H; q.y = qkv; q.ldy = 3 * H;
        launch_tc({q}, 1, r); }
      launch_attn(qkv, ao, L, H, &pao, r);
    }
    { TcSpec q; q.in = pao; q.w = L.t_o; q.bias = L.o.b; q.Cin = H; q.Cout = H; q.y = y; q.ldy = H;
      launch_tc({q}, 1, r); }
    klaunch(add_ln_kernel, lg, dim3(128), (size_t)0, x, y, L.ln1.g, L.ln1.b, (const float*)nullptr, (const float*)nullptr, 0, xb, tl, to, H, px1.hi, px1.lo, px1.mid);
    ++launches;
    { TcSpec q; q.in = px1; q.w = L.t_ffn1; q.bias = L.ffn1.b; q.Cin = H; q.Cout = Fc; q.k = ks; q.pad = (ks - 1) / 2;
      q.epi = TCE_RELU; q.out = pff; q.pl_slope = 1.f;
      launch_tc({q}, 1, r); }
    { TcSpec q; q.in = pff; q.w = L.t_ffn2; q.bias = L.ffn2.b; q.Cin = Fc; q.Cout = H; q.k = ks; q.pad = (ks - 1) / 2;
      q.y = y; q.ldy = H;
      launch_tc({q}, 1, r); }
    klaunch(add_ln_kernel, lg, dim3(128), (size_t)0, xb, y, L.ln2.g, L.ln2.b, (const float*)nullptr, va, cond_ld, x, tl, to, H, px.hi, px.lo, px.mid);
    ++launches;
  }
}

// Prior statistics m_p, logs_p (models.py:323-325): enc_p.proj of text_encoder's output -> d_stats [Ttok][2I].
void vtts_engine::prior_stats() {
  const int H = cfg.hidden_channels, I = cfg.inter_channels;
  const Rows r = tok_rows();
  float* stats = ensure(d_stats, (size_t)Ttok * 2 * I);
  if (enc_on_tc) {
    TcSpec q; q.in = enc_px; q.w = tc_encproj; q.bias = enc_proj.b; q.Cin = H; q.Cout = 2 * I; q.y = stats; q.ldy = 2 * I;
    launch_tc({q}, 1, r);
  } else {
    launch_conv({mk(enc_proj, d_x.p, H, 0, stats, 2 * I, 0, 1, 0)}, 1, r);
  }
}

// Token rows of a call (TTS phase 1, alignment): lengths and offsets of the token shape and, from host ids [B][t_max], the
// packed ids (zero between and behind the utterances), each checked against n_vocab.  ids null: packed on the device.
// phase1: room for phase 1's scalars, and speaker ids with host ids (filled by the caller); eps: for its noise (stage1).
void vtts_engine::stage_tokens(const int64_t* ids, int t_max, bool phase1, bool eps) {
  Staging& s = stg[STG_TOKENS];
  s.begin();
  s.add(d_tok_len, B);
  s.add(d_tok_off, B + 1);
  if (phase1) s.add(d_prm, 8);
  if (ids) s.add(d_ids, Ttok);
  if (ids && phase1) s.add(d_sid, B);
  if (eps) s.add(d_eps_dp, (size_t)B * 2 * maxTok);
  s.commit();
  memcpy(s.host(d_tok_len), h_tok_len.data(), B * sizeof(int));
  memcpy(s.host(d_tok_off), h_tok_off.data(), (B + 1) * sizeof(int));
  if (ids) {
    int* pi = s.host(d_ids);
    memset(pi, 0, (size_t)Ttok * sizeof(int));
    for (int b = 0; b < B; ++b)
      for (int t = 0; t < h_tok_len[b]; ++t) {
        const int64_t id = ids[(size_t)b * t_max + t];
        REQUIRE(id >= 0 && id < cfg.n_vocab, VTTS_ERR_INVALID, "phoneme id out of range [0, n_vocab)");
        pi[h_tok_off[b] + t] = (int)id;
      }
  }
}

// The phase-1 rest of the staging (after stage_tokens): scales and seed, the poll sequence (or without polling the frame
// lengths' readback), the speculation's frame cap and the duration predictor's noise.
void vtts_engine::stage1(int t_max, const float* noise_dp_host) {
  float* prm = stg[STG_TOKENS].host(d_prm);
  put_scalars(prm, 8, scales, 3, seed);
  if (!use_poll) {
    Staging& s = stg[STG_LENGTHS];
    s.begin();
    s.add(d_frm_len, B);
    s.add(d_frm_off, B + 1);
    s.commit();
  } else {
    const size_t need = (size_t)(2 * B + 4);
    if (need > map.cap) {
      REQUIRE(!capturing, VTTS_ERR_STATE, "mapped buffer growth during capture");
      if (map.p) CK(cudaStreamSynchronize(stream));
      CK(map.alloc(need + 256));
      map.p[0] = 0;
      ++ws_gen;
    }
    call_seq = (call_seq % 1000000) + 1;
    memcpy(&prm[6], &call_seq, 4);          // (0 without polling)
  }
  memcpy(&prm[7], &spec_cap, 4);           // frames the speculative second phase is sized for (0: none), see duration_kernel
  if (noise_dp_host) {        // [B][2][t_max] -> [B][2][maxTok]: the device layout depends on the length bucket only
    float* eps = stg[STG_TOKENS].host(d_eps_dp);
    for (int r = 0; r < 2 * B; ++r)
      memcpy(eps + (size_t)r * maxTok, noise_dp_host + (size_t)r * t_max, (size_t)std::min(t_max, maxTok) * sizeof(float));
    eps_dp_ld = maxTok;
  }
}

void vtts_engine::finish1() {
  if (use_poll) {
    // spin on the flag the last phase-1 kernel writes into mapped host memory (bounded; then fall back to a sync)
    volatile int* flag = map.p;
    bool seen = false;
    for (long spin = 0; spin < 40000000L; ++spin) {
      if (*flag == call_seq) { seen = true; break; }
      if ((spin & 0xFFFFF) == 0xFFFFF && cudaStreamQuery(stream) != cudaErrorNotReady) break;   // finished or failed
    }
    if (!seen) {
      CK(cudaStreamSynchronize(stream));
      REQUIRE(*flag == call_seq, VTTS_ERR_CUDA, "phase 1 finished without publishing the utterance lengths");
    }
    read_published_lengths();
    set_frame_shape();
    have_durations = true;
    return;
  }
  CK(cudaStreamSynchronize(stream));
  const int *len = stg[STG_LENGTHS].host(d_frm_len), *off = stg[STG_LENGTHS].host(d_frm_off);
  h_frm_len.assign(len, len + B);
  h_frm_off.assign(off, off + B + 1);
  check_frame_lengths(h_frm_len.data(), h_frm_off[B], B);
  set_frame_shape();
  have_durations = true;
}

// ---------------------------------------------------------------------------------------------------
// Phase 2: alignment + prior sampling, flow^-1, decoder.
// ---------------------------------------------------------------------------------------------------
void vtts_engine::phase2(const float* noise_z, int z_ld, bool noise_on_device, bool run_decoder) {
  const vtts_config& c = cfg;
  const int H = c.hidden_channels, I = c.inter_channels, half = I / 2;
  const size_t F = (size_t)Tfrm;
  const int* tl = d_tok_len.p;
  const int* to = d_tok_off.p;
  const int* fl = d_frm_len.p;
  const int* fo = d_frm_off.p;
  const Rows r = frm_rows();
  if (!capturing) CK(cudaEventRecord(ev[4], stream));
  if (noise_z && !noise_on_device) {
    // host noise was staged by the caller (stage_noise_z) as [B][I][maxFrm]: the layout depends on the bucket only
    stg[STG_NOISE_Z].upload();
    noise_z = d_eps_z.p;
    z_ld = maxFrm;
  }
  float* z = ensure(d_z, F * I);
  int* ftok = ensure(d_ftok, F);
  {
    dim3 g(maxFrm, B);
    klaunch(sample_prior_kernel, dim3(g), dim3(64), (size_t)(0), d_stats.p, I, d_cum.p, tl, to, fl, fo, noise_z, z_ld, d_prm.p, z, ftok);
    CK(cudaGetLastError());
    ++launches;
  }
  if (debug_flags & 1) {
    float* zp = ensure(d_zp_dbg, F * I);
    CK(cudaMemcpyAsync(zp, z, F * I * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  }
  // ---- flow, reverse (models.py:750-757).  Flip (modules.py:272-279) is folded into the packed pre/post
  // weights: for a "flipped" layer x0 lives in physical channels [half, 2*half), x1 in [0, half).
  float* h = ensure(d_h, F * H);
  float* h1 = ensure(d_h1, F * H);
  float* wx = ensure(d_wx, F * H);
  float* acts = ensure(d_acts, F * H);
  float* skip = ensure(d_skip, F * H);
  float* fy = ensure(d_fy, F * H);
  float* fqkv = nullptr; float* fao = nullptr; float* ffh2 = nullptr;
  if (c.use_transformer_flows) {
    fqkv = ensure(d_fqkv, F * 3 * H);
    fao = ensure(d_fao, F * H);
    ffh2 = ensure(d_ffh2, F * H);
  }
  const int nf = c.flow_n_flows, nl = c.flow_wn_layers, fk = c.flow_kernel_size;
  const bool flow_on_tc = tc && !flow.empty() && !flow[0].t_in.empty();
  const bool dec_now = tc && run_decoder;
  const bool emit_pz = flow_on_tc && dec_now && nf >= 2 && !(debug_flags & 2);
  if (flow_on_tc || dec_now) {
    begin_planes();
    if (flow_on_tc) alloc_flow_planes();
    if (dec_now) alloc_decoder_planes();
    flush_tails(fl, fo);
  }
  (void)h; (void)h1; (void)wx; (void)acts; (void)skip; (void)fy; (void)fqkv; (void)fao; (void)ffh2; (void)nl; (void)fk; (void)half;
  const float* cond = has_g ? d_condv.p : nullptr;
  if (flow_on_tc) flow_tc(z, emit_pz, cond, condR, /*forward=*/false, r);
  else flow_ffma(z, cond, condR, /*forward=*/false, r);
  if (!capturing) CK(cudaEventRecord(ev[5], stream));

  if (!run_decoder) return;
  decode(z, r, /*planes_ready=*/dec_now, /*pz_ready=*/emit_pz);
}

// Flow on the fp32 pipe (models.py:750-757).  Flip (modules.py:272-279) is folded into the packed pre/post weights: for a
// "flipped" layer x0 lives in physical channels [half, 2*half), x1 in [0, half).  forward / cond: see flow_tc.
void vtts_engine::flow_ffma(float* z, const float* cond, int cond_ld, bool forward, const Rows& r) {
  const vtts_config& c = cfg;
  const int H = c.hidden_channels, I = c.inter_channels, half = I / 2;
  const size_t F = (size_t)Tfrm;
  float* h = ensure(d_h, F * H);
  float* h1 = ensure(d_h1, F * H);
  float* wx = ensure(d_wx, F * H);
  float* acts = ensure(d_acts, F * H);
  float* skip = ensure(d_skip, F * H);
  float* fy = ensure(d_fy, F * H);
  float* fqkv = nullptr; float* fao = nullptr; float* ffh2 = nullptr;
  if (c.use_transformer_flows) {
    fqkv = ensure(d_fqkv, F * 3 * H);
    fao = ensure(d_fao, F * H);
    ffh2 = ensure(d_ffh2, F * H);
  }
  const int nf = c.flow_n_flows, nl = c.flow_wn_layers, fk = c.flow_kernel_size;
  for (int s = 0; s < nf; ++s) {
    const int f = forward ? s : nf - 1 - s;
    const FlowW& W = flow[f];
    const bool flipped = ((nf - f) % 2) == 1;
    const int x0off = flipped ? half : 0, x1off = flipped ? 0 : half;
    launch_conv({mk(W.pre, z, I, x0off, h, H, 0, 1, 0)}, 1, r);
    float* wn_in = h;
    if (c.use_transformer_flows) {
      // h = h + Encoder(h)  (models.py:377): the layer's last LN adds `h` back and lands in wx
      float* xa = h; float* xb2 = h1;
      // encoder_layer writes its result into `xa` (== h) -- we need h preserved for the residual, so run the
      // layer on explicit buffers instead of the ping-pong helper:
      launch_conv({mk(W.tr.qkv, h, H, 0, fqkv, 3 * H, 0, 1, 0)}, 1, r);
      launch_attn(fqkv, fao, W.tr, H, nullptr, r);
      launch_conv({mk(W.tr.o, fao, H, 0, fy, H, 0, 1, 0)}, 1, r);
      dim3 lg((r.maxLen + 3) / 4, r.n);
      klaunch(add_ln_kernel, dim3(lg), dim3(128), (size_t)(0), xa, fy, W.tr.ln1.g, W.tr.ln1.b, nullptr, nullptr, 0, xb2, r.lens, r.offs, H, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr);
      CK(cudaGetLastError());
      ++launches;
      {
        ConvP p = mk(W.tr.ffn1, xb2, H, 0, ffh2, H, 0, 1, (fk - 1) / 2);
        p.epi = EPI_RELU;
        launch_conv({p}, 1, r);
      }
      launch_conv({mk(W.tr.ffn2, ffh2, H, 0, fy, H, 0, 1, (fk - 1) / 2)}, 1, r);
      klaunch(add_ln_kernel, dim3(lg), dim3(128), (size_t)(0), xb2, fy, W.tr.ln2.g, W.tr.ln2.b, h, nullptr, 0, wx, r.lens, r.offs, H, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr);
      CK(cudaGetLastError());
      ++launches;
      wn_in = wx;
    }
    // WN (modules.py:148-176).  The hidden state is updated in place in `wn_in`.
    wn_ffma(W.in, W.rsx, W.rss, nl, fk, c.flow_dilation_rate, wn_in, acts, skip, cond ? cond + r_flow + f * nl * 2 * H : nullptr, cond_ld, r);
    {
      // x1 <- x1 - post(h) (reverse) / x1 + post(h) (forward) (mean_only; models.py:381-391)
      ConvP p = mk(W.post, skip, H, 0, z, I, x1off, 1, 0);
      p.alpha = forward ? 1.f : -1.f;
      p.res = z; p.ldr = I; p.roff = x1off;
      launch_conv({p}, 1, r);
    }
  }
}

void vtts_engine::wn_ffma(const std::vector<ConvW>& in, const std::vector<ConvW>& rsx, const std::vector<ConvW>& rss, int nl, int fk,
                          int dil_rate, float* x, float* acts, float* skip, const float* cond, int cond_ld, const Rows& r) {
  const int H = cfg.hidden_channels;
  int dil = 1;
  for (int i = 0; i < nl; ++i) {
    {
      ConvP p = mk(in[i], x, H, 0, acts, H, 0, dil, dil * (fk - 1) / 2);
      p.epi = EPI_GATE;
      if (cond) { p.cond = cond + i * 2 * H; p.cond_ld = cond_ld; }
      launch_conv({p}, 1, r);
    }
    ConvP ps = mk(rss[i], acts, H, 0, skip, H, 0, 1, 0);
    if (i > 0) { ps.res = skip; ps.ldr = H; ps.roff = 0; }
    if (i < nl - 1) {
      ConvP px = mk(rsx[i], acts, H, 0, x, H, 0, 1, 0);
      px.res = x; px.ldr = H; px.roff = 0;
      launch_conv({px, ps}, 1, r);
    } else {
      launch_conv({ps}, 1, r);
    }
    dil *= dil_rate;
  }
}

// Decoder over the rows r -- the whole batch, or one halo-extended chunk of a single
// utterance (vtts_decode_chunk).
void vtts_engine::decode(float* z, const Rows& r, bool planes_ready, bool pz_ready) {
  const vtts_config& c = cfg;
  const int I = c.inter_channels;
  const size_t F = (size_t)Tfrm;
  // ---- decoder (models.py:1016-1054 / 872-891)
  int ch = c.upsample_initial_channel, rm = 1, i0 = 0;
  float* cur = nullptr;
  if (tc) {
    if (!planes_ready) {          // (chunked decoding: the decoder runs on its own)
      begin_planes();
      alloc_decoder_planes();
      flush_tails(r.lens, r.offs);
    }
    if (decoder_tc(z, pz_ready, r)) {
      if (!capturing) CK(cudaEventRecord(ev[6], stream));
      return;
    }
    // the vocoder: stages voc_nt.. on the FFMA pipe, from the upsampled rows decoder_tc left in d_stage[voc_nt]
    i0 = voc_nt;
    for (int i = 0; i < i0; ++i) { rm *= c.upsample_rates[i]; ch /= 2; }
  } else {
    cur = ensure(d_d0, F * ch);
    ConvP p = mk(dec_pre, z, I, 0, cur, ch, 0, 1, 3);
    if (r_dec >= 0) { p.cond = d_condv.p + r_dec; p.cond_ld = condR; }     // x = conv_pre(z) + cond(g)
    launch_conv({p}, 1, r);
  }
  const int nk = c.n_resblock_kernels, nd = c.n_resblock_dilations;
  if ((int)d_stage.size() < c.n_upsamples) {
    d_stage.resize(c.n_upsamples);
    d_xj.resize(c.n_upsamples);
    d_tmp.resize(c.n_upsamples);
    for (int i = 0; i < c.n_upsamples; ++i) { d_xj[i].resize(nk); d_tmp[i].resize(nk); }
  }
  for (int i = i0; i < c.n_upsamples; ++i) {
    const int u = c.upsample_rates[i], ch2 = ch / 2;
    const size_t rows = F * rm * u;
    float* X = ensure(d_stage[i], rows * ch2);
    for (int r0 = 0; r0 < u && cur; r0 += CV_MAXP) {
      std::vector<ConvP> ps;
      for (int ph = r0; ph < std::min(u, r0 + CV_MAXP); ++ph) {
        ConvP p = mk(ups[i].phase[ph], cur, ch, 0, X, ch2, 0, 1, ups[i].pad[ph]);
        p.pro = PRO_LRELU; p.slope = 0.1f;
        p.out_mul = u; p.out_add = ph;
        ps.push_back(p);
      }
      launch_conv(ps, rm, r);
    }
    rm *= u;
    ch = ch2;
    std::vector<float*> xj(nk), tmp(nk);
    for (int j = 0; j < nk; ++j) {
      xj[j] = ensure(d_xj[i][j], rows * ch);
      tmp[j] = ensure(d_tmp[i][j], rows * ch);
    }
    for (int d = 0; d < nd; ++d) {
      std::vector<ConvP> p1, p2;
      for (int j = 0; j < nk; ++j) {
        const RbW& R = rbs[i * nk + j];
        const int k = c.resblock_kernel_sizes[j], dl = c.resblock_dilations[j][d];
        const float* src = (d == 0) ? X : xj[j];
        if (c.resblock_type == 1) {
          ConvP a = mk(R.c1[d], src, ch, 0, tmp[j], ch, 0, dl, dl * (k - 1) / 2);
          a.pro = PRO_LRELU; a.slope = 0.1f;
          ConvP b2 = mk(R.c2[d], tmp[j], ch, 0, xj[j], ch, 0, 1, (k - 1) / 2);
          b2.pro = PRO_LRELU; b2.slope = 0.1f;
          b2.res = src; b2.ldr = ch; b2.roff = 0;
          p1.push_back(a);
          p2.push_back(b2);
        } else {
          ConvP a = mk(R.c1[d], src, ch, 0, (d == 0) ? xj[j] : tmp[j], ch, 0, dl, dl * (k - 1) / 2);
          a.pro = PRO_LRELU; a.slope = 0.1f;
          a.res = src; a.ldr = ch; a.roff = 0;
          p1.push_back(a);
        }
      }
      launch_conv(p1, rm, r);
      if (c.resblock_type == 1) {
        launch_conv(p2, rm, r);
      } else if (d > 0) {
        for (int j = 0; j < nk; ++j) std::swap(xj[j], tmp[j]);   // ResBlock2 ping-pong (halo reads forbid in-place)
      }
    }
    mrf_mean(xj, X, (long)(rows * ch / 4));
    cur = X;
  }
  float* wav = ensure(d_wav, F * hop + 16);
  if (c.decoder_type == 0) {
    const int cps = c.istft_n_fft + 2, pc = c.subbands * cps;
    float* post = ensure(d_post, (F * rm + B) * pc);
    ConvP p = mk(dec_post, cur, ch, 0, post, pc, 0, 1, 3);
    p.pro = PRO_LRELU; p.slope = 0.01f;
    p.reflect = 1; p.in_extra = 1; p.out_seq_extra = 1;
    launch_conv({p}, rm, r);
    istft_tail(post, rm, r, wav);
  } else {
    ConvP p = mk(dec_post, cur, ch, 0, wav, 1, 0, 1, 3);
    p.pro = PRO_LRELU; p.slope = 0.01f;
    p.epi = EPI_TANH;
    launch_conv({p}, rm, r);
  }
  if (!capturing) CK(cudaEventRecord(ev[6], stream));
}

// ---------------------------------------------------------------------------------------------------
// Voice conversion (models.py:1710-1718): spectrogram front end, enc_q with g_src, flow forward with g_src, flow reverse
// with g_tgt, decoder.  The frame counts follow from the input lengths, so the whole call is ONE graphed phase.
// ---------------------------------------------------------------------------------------------------
// Staged inputs of a call on recordings (voice conversion, alignment, speaker embedding, QuickVC conversion): frame lengths
// and offsets, d_vint [clip_len B][sid_src B][sid_tgt B], the per-call scalars, the input (wav [B][vc_wld], spec
// [B][C][maxFrm], unit rows [Tfrm][QV_UNITS] packed as the engine's rows, or none), g [B][gin] (QuickVC conversion only) and
// the posterior eps [B][inter][maxFrm].
void vtts_engine::stage_clip_fields(ClipIn in, bool eps) {
  const vtts_config& c = cfg;
  Staging& s = stg[STG_CLIPS];
  s.begin();
  s.add(d_frm_len, B);
  s.add(d_frm_off, B + 1);
  s.add(d_vint, 3 * B);
  s.add(d_vprm, 16);
  if (in == IN_WAV) s.add(d_vin, (size_t)B * vc_wld);
  if (in == IN_SPEC) s.add(d_vin, (size_t)B * c.spec_channels * maxFrm);
  if (in == IN_UNITS) s.add(d_vin, (size_t)Tfrm * QV_UNITS);
  if (in >= IN_UNITS) s.add(d_qg, (size_t)B * c.gin_channels);
  if (eps) s.add(d_vnoise, (size_t)B * c.inter_channels * maxFrm);
  s.commit();
}

// Uploads the staged inputs of a call on recordings (stage_clip_fields); returns the posterior eps (null: Philox).
float* vtts_engine::vc_upload(bool eps) {
  stg[STG_CLIPS].upload();
  return eps ? d_vnoise.p : nullptr;
}

// Conditioning rows of g_src (rows [0, condR) of the stacked TTS matrix, then enc_q's q_R rows) -> d_vcsrc [B][condR + q_R];
// with `tgt` also g_tgt's TTS rows -> d_condv [B][condR], in the same launch (cond_vc_kernel, sid from d_vint).
float* vtts_engine::cond_src(bool tgt) {
  const int qld = condR + q_R;
  float* csrc = ensure(d_vcsrc, (size_t)B * qld);
  float* ctgt = tgt ? ensure(d_condv, (size_t)B * condR) : nullptr;
  klaunch(cond_vc_kernel, dim3((qld + 7) / 8, tgt ? 2 * B : B), dim3(256), (size_t)(cfg.gin_channels * sizeof(float)), emb_g,
          (const int*)(d_vint.p + B), cond_w, cond_b, condR, q_cond_w, q_cond_b, q_R, csrc, ctgt, cfg.gin_channels, B, cfg.n_speakers);
  CK(cudaGetLastError());
  ++launches;
  return csrc;
}

// Front end, posterior encoder and forward flow (models.py:836-842, 750-753): the uploaded waveform / spectrogram -> z
// (vc_z) -> z_p = flow(z, g_src) in d_z.  csrc: g_src's rows [B][condR + q_R] (cond_src), null for an unconditioned model.
// Opens the phase's plane collection (the flow's WN planes, also used by enc_q) for the frame shape.
// Spectrogram front end of the uploaded waveforms (vc_upload) -> feature rows [Tfrm][spec_pad] (d_vfeat): the magnitude
// spectrogram, or its log-mel when the model reads mel; caller-supplied features are only repacked.
float* vtts_engine::front_end(bool from_spec) {
  const vtts_config& c = cfg;
  const size_t F = (size_t)Tfrm;
  const int* fl = d_frm_len.p;
  const int* fo = d_frm_off.p;
  const int* vi = d_vint.p;
  const float* vin = d_vin.p;
  float* feat = ensure(d_vfeat, F * spec_pad);
  if (from_spec) {
    klaunch(spec_pack_kernel, dim3(maxFrm, B), dim3(128), (size_t)0, vin, c.spec_channels, maxFrm, fl, fo, feat, spec_pad);
    CK(cudaGetLastError());
    ++launches;
  } else {
    const int nbins = c.filter_length / 2 + 1;
    const bool mel = c.use_mel_posterior_encoder != 0;
    float* lin = mel ? ensure(d_vlin, F * nbins) : feat;
    dim3 g((maxFrm + ST_TM - 1) / ST_TM, c.filter_length / ST_TN, B);
    klaunch(stft_mag_kernel, g, dim3(ST_THREADS), (size_t)0, vin, (long)vc_wld, vi, stft_basis, c.filter_length,
            c.hop_length, vc_pad, fl, fo, lin, mel ? nbins : spec_pad);
    CK(cudaGetLastError());
    ++launches;
    if (mel) {
      klaunch(mel_log_kernel, dim3((maxFrm + MEL_ROWS - 1) / MEL_ROWS, B), dim3(MEL_THREADS), (size_t)MEL_ROWS * nbins * sizeof(float),
              (const float*)lin, nbins, mel_fb, nbins, c.n_mel_channels, fl, fo, feat, spec_pad);
      CK(cudaGetLastError());
      ++launches;
    }
  }
  return feat;
}

// Posterior encoder over feature rows [Tfrm][feat_ld] (models.py:836-842; QuickVC's enc_p, vc/models.py:264-271): pre ->
// 16-layer WN (cond rows qcond, row stride qld; null: none) -> proj -> stats (d_vstats) -> z = m + eps * exp(logs) in d_z.
// Opens the phase's plane collection (the flow's WN planes, also used here) for the frame shape.
void vtts_engine::posterior_encode(const float* feat, int feat_ld, const float* noise, const float* qcond, int qld, const Rows& r) {
  const vtts_config& c = cfg;
  const int H = c.hidden_channels, I = c.inter_channels;
  const size_t F = (size_t)Tfrm;
  float* h = ensure(d_h, F * H);
  float* acts = ensure(d_acts, F * H);
  float* skip = ensure(d_skip, F * H);
  float* stats = ensure(d_vstats, F * 2 * I);
  float* z = ensure(d_z, F * I);
  const bool flow_on_tc = tc && !flow.empty() && !flow[0].t_in.empty();
  if (flow_on_tc || q_tc) {
    begin_planes();
    alloc_flow_planes();                     // (enc_q uses the flow's WN planes before the flow runs)
    flush_tails(r.lens, r.offs);
  }
  {
    ConvP p = mk(q_pre, feat, feat_ld, 0, h, H, 0, 1, 0);
    if (q_tc) { p.p_hi = flp.pwx.hi; p.p_lo = flp.pwx.lo; p.ldp = H; p.pl_slope = 1.f; }
    launch_conv({p}, 1, r);
  }
  if (q_tc) {
    wn_tc(qt_in, q_in, qt_rsx, q_rsx, qt_rss, q_rss, Q_LAYERS, Q_KERNEL, 1, h, skip, flp.pwx, flp.pacts, flp.pskip, qcond, qld, r);
    TcSpec q; q.in = flp.pskip; q.w = qt_proj; q.bias = q_proj.b; q.Cin = H; q.Cout = 2 * I; q.y = stats; q.ldy = 2 * I;
    launch_tc({q}, 1, r);
  } else {
    wn_ffma(q_in, q_rsx, q_rss, Q_LAYERS, Q_KERNEL, 1, h, acts, skip, qcond, qld, r);
    launch_conv({mk(q_proj, skip, H, 0, stats, 2 * I, 0, 1, 0)}, 1, r);
  }
  klaunch(posterior_sample_kernel, dim3(r.maxLen, r.n), dim3(64), (size_t)0, (const float*)stats, I, noise, maxFrm,
          (const float*)d_vprm.p, r.lens, r.offs, z);
  CK(cudaGetLastError());
  ++launches;
  if (debug_flags & 1) CK(cudaMemcpyAsync(ensure(d_vz_dbg, F * I), z, F * I * sizeof(float), cudaMemcpyDeviceToDevice, stream));
}

void vtts_engine::posterior_side(bool from_spec, const float* noise, const float* csrc, const Rows& r) {
  const int I = cfg.inter_channels;
  const size_t F = (size_t)Tfrm;
  const int qld = condR + q_R;
  // ---- enc_q input rows [F][spec_pad]
  float* feat = front_end(from_spec);
  // ---- posterior encoder (models.py:836-842): pre -> 16-layer WN (g_src) -> proj -> sample
  posterior_encode(feat, spec_pad, noise, csrc ? csrc + condR : nullptr, qld, r);
  float* z = d_z.p;
  // ---- z_p = flow(z, g_src)   (models.py:1715, 1640)
  const bool flow_on_tc = tc && !flow.empty() && !flow[0].t_in.empty();
  if (flow_on_tc) flow_tc(z, false, csrc, qld, /*forward=*/true, r);
  else flow_ffma(z, csrc, qld, /*forward=*/true, r);
  if (debug_flags & 1) CK(cudaMemcpyAsync(ensure(d_vzp_dbg, F * I), z, F * I * sizeof(float), cudaMemcpyDeviceToDevice, stream));
}

void vtts_engine::convert_enqueue(bool from_spec, bool eps) {
  if (!capturing) CK(cudaEventRecord(ev[4], stream));
  const float* noise = vc_upload(eps);
  const Rows r = frm_rows();
  // ---- g_src / g_tgt (models.py:1712-1713) and every cond row of both, one launch: src -> d_vcsrc [B][condR + q_R]
  //      (the TTS rows, then enc_q's), tgt -> d_condv [B][condR] (where the reverse flow and the decoder read them)
  const float* csrc = cond_src(/*tgt=*/true);
  const float* ctgt = d_condv.p;
  posterior_side(from_spec, noise, csrc, r);
  // ---- z_hat = flow^-1(z_p, g_tgt)   (models.py:1716)
  float* z = d_z.p;
  const bool flow_on_tc = tc && !flow.empty() && !flow[0].t_in.empty();
  if (flow_on_tc) flow_tc(z, false, ctgt, condR, /*forward=*/false, r);
  else flow_ffma(z, ctgt, condR, /*forward=*/false, r);
  if (!capturing) CK(cudaEventRecord(ev[5], stream));
  // ---- o_hat = dec(z_hat * y_mask, g=g_tgt)   (models.py:1717)
  decode(z, r);
}

// ---------------------------------------------------------------------------------------------------
// Forced alignment: the text-to-frame alignment at the head of SynthesizerTrn.forward (models.py:1632-1660) -- enc_p on the
// ids, enc_q + forward flow on the recording (g_src; none for a single-speaker model), neg_cent, MAS -- as ONE graphed phase.
// Token lengths come from the input and frame lengths from the clip lengths, so nothing waits for the host.  The
// noise-scaled MAS of :1653-1655 is a training regulariser (off in the shipped configuration) and is never added here.
// ---------------------------------------------------------------------------------------------------
void vtts_engine::align_enqueue(bool from_spec, bool eps) {
  const int I = cfg.inter_channels;
  if (!capturing) CK(cudaEventRecord(ev[0], stream));
  const float* noise = vc_upload(eps);
  stg[STG_TOKENS].upload();                         // (staged by the host: lengths, offsets, packed ids)
  const int* tl = d_tok_len.p;
  const int* to = d_tok_off.p;
  const int* fl = d_frm_len.p;
  const int* fo = d_frm_off.p;
  const float* csrc = has_g ? cond_src(/*tgt=*/false) : nullptr;
  // ---- m_p, logs_p = enc_p(x, g)   (models.py:1632-1633)
  text_encoder(csrc, condR + q_R);
  prior_stats();
  if (!capturing) CK(cudaEventRecord(ev[2], stream));
  // ---- z_p = flow(enc_q(y, g), g)   (models.py:1639-1640)
  posterior_side(from_spec, noise, csrc, frm_rows());
  if (!capturing) CK(cudaEventRecord(ev[4], stream));
  // ---- neg_cent [B][T_y][T_x] over the frame and token buckets (models.py:1645-1651), then MAS (:1656-1660)
  const int Ty = maxFrm, Tx = maxTok;
  float* nc = ensure(d_ncent, (size_t)B * Ty * Tx);
  if (debug_flags & 1) CK(cudaMemsetAsync(nc, 0xFF, (size_t)B * Ty * Tx * sizeof(float), stream));   // NaN outside the utterances
  klaunch(neg_cent_kernel, dim3((Tx + NC_T - 1) / NC_T, (Ty + NC_T - 1) / NC_T, B), dim3(NC_THREADS), (size_t)0, (const float*)d_z.p,
          (const float*)d_stats.p, I, fl, fo, tl, to, nc, Ty, Tx);
  CK(cudaGetLastError());
  ++launches;
  if (debug_flags & 1) {       // [B][max t_y][max t_x] (debug runs are eager: the real shape is known here)
    float* dbg = ensure(d_ncent_dbg, (size_t)B * real_maxFrm * real_maxTok);
    for (int b = 0; b < B; ++b)
      CK(cudaMemcpy2DAsync(dbg + (size_t)b * real_maxFrm * real_maxTok, (size_t)real_maxTok * sizeof(float), nc + (size_t)b * Ty * Tx,
                           (size_t)Tx * sizeof(float), (size_t)real_maxTok * sizeof(float), real_maxFrm, cudaMemcpyDeviceToDevice, stream));
  }
  int* dur = ensure(d_adur, Ttok);
  int* tof = ensure(d_atof, Tfrm);
  float* score = ensure(d_ascore, B);
  klaunch(mas_kernel, dim3(B), dim3(MAS_THREADS), (size_t)2 * Tx * sizeof(float), nc, (int*)nullptr, fl, tl, Ty, Tx, tof, fo, dur, to,
          score);
  CK(cudaGetLastError());
  ++launches;
  if (!capturing) CK(cudaEventRecord(ev[5], stream));
}

// ---------------------------------------------------------------------------------------------------
// QuickVC speaker encoder (SpeakerEncoder.embed_utterance, vc/models.py:728-767).  A QuickVC blob (weights.pack_quickvc) holds
// the encoder and the mel front end; none of the VITS2 tensors.
// ---------------------------------------------------------------------------------------------------
void vtts_engine::bind_quickvc() {
  const vtts_config& c = cfg;
  REQUIRE(c.gin_channels == SPK_H, VTTS_ERR_INVALID, "the speaker encoder needs gin_channels == 256 (its LSTM hidden size)");
  REQUIRE(c.n_mel_channels % CV_CK == 0 && c.spec_channels == c.n_mel_channels && c.use_mel_posterior_encoder, VTTS_ERR_INVALID,
          "the speaker encoder reads n_mel_channels (a multiple of 16) log-mel rows");
  REQUIRE(c.filter_length > 0 && c.hop_length > 0 && c.filter_length % ST_TN == 0 && c.filter_length > c.hop_length &&
              (c.filter_length - c.hop_length) % 2 == 0 && c.win_length == c.filter_length,
          VTTS_ERR_INVALID, "bad spectrogram configuration (filter_length must be a multiple of 64, above hop_length, == win_length)");
  REQUIRE(mel_smem_bytes(c.filter_length) <= (size_t)MEL_SMEM_MAX, VTTS_ERR_INVALID,
          "filter_length too large for the mel projection (its spectrum rows must fit in shared memory)");
  spec_pad = c.n_mel_channels;
  vc_pad = (c.filter_length - c.hop_length) / 2;
  for (int l = 0; l < 3; ++l) {
    const std::string p = "spk.l" + std::to_string(l);
    spk_ih[l] = conv(p + ".ih", l == 0 ? c.n_mel_channels : SPK_H, SPK_GATES, 1);
    spk_hh[l] = vec(p + ".hh", (size_t)SPK_GATES * SPK_H);
  }
  spk_lin_w = vec("spk.lin.w", (size_t)SPK_H * SPK_H);
  spk_lin_b = vec("spk.lin.b", SPK_H);
  stft_basis = vec("vc.stft", (size_t)c.filter_length * c.filter_length);
  mel_fb = vec("vc.mel", (size_t)c.n_mel_channels * (c.filter_length / 2 + 1));
  // clusters that fit at once: a cluster must sit inside one GPC, so this can be fewer than n_sm / SPK_CTAS
  auto fit = [&](auto kern, size_t smem, int& out) {
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t lc;
    memset(&lc, 0, sizeof(lc));
    lc.gridDim = dim3(SPK_CTAS * 64); lc.blockDim = dim3(SPK_THREADS); lc.dynamicSmemBytes = smem;
    int nc = 0;
    if (cudaOccupancyMaxActiveClusters(&nc, kern, &lc) != cudaSuccess) { nc = 0; cudaGetLastError(); }
    out = std::max(1, nc);
  };
  fit(lstm_rec_kernel<1>, spk_rec_smem<1>(), spk_clusters[0]);
  fit(lstm_rec_kernel<2>, spk_rec_smem<2>(), spk_clusters[1]);
  fit(lstm_rec_kernel<4>, spk_rec_smem<4>(), spk_clusters[2]);
  fit(lstm_rec_kernel<8>, spk_rec_smem<8>(), spk_clusters[3]);
  // ---- the conversion side, when the blob has it (weights.pack_quickvc of a whole checkpoint)
  has_encp = tensors.count("encp.pre.b") > 0;
  if (has_encp) {
    REQUIRE(c.decoder_type == 0 && c.resblock_type == 1 && c.n_upsamples == 2 && !c.use_transformer_flows && c.flow_n_flows % 2 == 0 &&
                c.hidden_channels % 32 == 0 && c.hidden_channels <= 256 && c.n_resblock_kernels <= CV_MAXP,
            VTTS_ERR_INVALID, "unsupported QuickVC configuration (the published ms_istft_vits model: two upsampling stages, "
            "ResBlock1, plain coupling flow with an even number of layers)");
    r_flow = 0;
    r_dec = c.flow_n_flows * c.flow_wn_layers * 2 * c.hidden_channels;
    condR = r_dec + c.upsample_initial_channel;
    cond_w = vec("cond.w", (size_t)condR * c.gin_channels);
    cond_b = vec("cond.b", condR);
    bind_flow_decoder();
    bind_wn_encoder("encp", QV_UNITS);
    istft_w2 = vec("dec.w2", (size_t)c.istft_n_fft);
  }
  bind_contentvec();
}

void vtts_engine::bind_contentvec() {
  const vtts_config& c = cfg;
  has_cv = c.cv_layers > 0 && tensors.count("cv.c0.w") > 0;
  if (!has_cv) return;
  const int NL = c.cv_n_conv, C = c.cv_conv_dim, H = c.cv_hidden, Fh = c.cv_ffn, G = c.cv_pos_groups;
  REQUIRE(NL >= 2 && NL <= 8 && C % CV_CK == 0 && C <= 32 * CVL_MAXV && c.cv_conv_kernel[0] >= 1 && c.cv_conv_kernel[0] <= CVG_KMAX &&
              c.cv_conv_stride[0] >= 1,
          VTTS_ERR_INVALID, "unsupported ContentVec feature encoder (2..8 convs, width a multiple of 16 up to 1024, layer 0 up to 16 taps)");
  cv_P = 1;
  for (int i = 1; i < NL; ++i) {
    REQUIRE(c.cv_conv_kernel[i] >= 1 && c.cv_conv_stride[i] >= 1, VTTS_ERR_INVALID, "bad ContentVec conv kernel / stride");
    cv_P *= c.cv_conv_stride[i];
  }
  REQUIRE(cv_P <= 4096, VTTS_ERR_INVALID, "ContentVec strides too large");
  REQUIRE(H % c.cv_heads == 0 && (H / c.cv_heads) % 32 == 0 && H / c.cv_heads <= 128 && H <= 32 * CVL_MAXV && Fh % CV_CK == 0,
          VTTS_ERR_INVALID, "unsupported ContentVec transformer (head width a multiple of 32 up to 128, width up to 1024)");
  REQUIRE(G >= 1 && H % G == 0 && (H / G) % CV_CK == 0 && c.cv_pos_k % 2 == 0 && CV_TT + c.cv_pos_k / 2 - 1 <= 32 * CV_XR, VTTS_ERR_INVALID,
          "unsupported ContentVec positional conv (even kernel up to 130, group width a multiple of 16)");
  const int K0 = c.cv_conv_kernel[0], kh = c.cv_pos_k / 2, Cg = H / G;
  cv_w0 = vec("cv.c0.w", (size_t)C * K0);
  cv_gn_g = vec("cv.gn.g", C);
  cv_gn_b = vec("cv.gn.b", C);
  for (int i = 1; i < NL; ++i) cv_conv[i] = conv("cv.c" + std::to_string(i), c.cv_conv_kernel[i] * C, C, 1);
  cv_fp_g = vec("cv.fp.ln.g", C);
  cv_fp_b = vec("cv.fp.ln.b", C);
  cv_fp = conv("cv.fp", C, H, 1);
  cv_pos_w = vec("cv.pos.w", (size_t)2 * G * kh * Cg * Cg);
  cv_pos_b = vec("cv.pos.b", H);
  cv_enc_g = vec("cv.enc.ln.g", H);
  cv_enc_b = vec("cv.enc.ln.b", H);
  // zeros: the bias of the positional conv's second half, the relative tables (fp32, and the [16][128] bf16 tiles of the
  // tensor-core attention)
  const size_t nz = std::max<size_t>({(size_t)H, (size_t)(2 * c.window_size + 1) * (H / c.cv_heads), (size_t)ATC_RELP * 128});
  float* zero = ensure(d_cvzero, nz);
  CK(cudaMemsetAsync(zero, 0, d_cvzero.cap * sizeof(float), stream));
  cv_tc = c.precision >= 1 && c.precision <= 3;
  if (cv_tc) {
    REQUIRE(C % TC_BK == 0 && H % TC_BK == 0 && Fh % TC_BK == 0 && 2 * c.window_size + 1 <= ATC_RELP, VTTS_ERR_INVALID,
            "ContentVec on the tensor cores needs widths in multiples of 64");
    REQUIRE(tensors.count("cv.fp.th") > 0, VTTS_ERR_WEIGHTS, "the blob lacks ContentVec's tensor-core weights (packed with precision 0)");
    cv_tfp = tcw("cv.fp", C, H, 1);
  }
  cv_enc.clear();
  for (int l = 0; l < c.cv_layers; ++l) {
    const std::string p = "cv.l" + std::to_string(l);
    EncLayerW L;
    L.heads = c.cv_heads;
    L.qkv = conv(p + ".qkv", H, 3 * H, 1);
    L.o = conv(p + ".o", H, H, 1);
    L.ln1 = ln(p + ".ln1", H);
    L.ffn1 = conv(p + ".ffn1", H, Fh, 1);
    L.ffn2 = conv(p + ".ffn2", Fh, H, 1);
    L.ln2 = ln(p + ".ln2", H);
    L.relk = L.relv = zero;
    if (cv_tc) {
      L.t_qkv = tcw(p + ".qkv", H, 3 * H, 1);
      L.t_o = tcw(p + ".o", H, H, 1);
      L.t_ffn1 = tcw(p + ".ffn1", H, Fh, 1);
      L.t_ffn2 = tcw(p + ".ffn2", Fh, H, 1);
      const __nv_bfloat16* zb = reinterpret_cast<const __nv_bfloat16*>(zero);
      L.rk_hi = L.rk_lo = L.rv_hi = L.rv_lo = zb;
    }
    cv_enc.push_back(L);
  }
}

// Host side of a ContentVec call: every level's lengths and offsets follow from the sample counts, so nothing waits for the
// device.  Clip b's layer-0 rows start at a multiple of cv_P (so every later level's offset is an exact division) and its
// samples are staged at s0 times that row.  Returns each clip's frame count.
std::vector<int> vtts_engine::cv_stage(const float* wav, const int64_t* lengths, int64_t ld) {
  const vtts_config& c = cfg;
  const int NL = c.cv_n_conv, K0 = c.cv_conv_kernel[0], s0 = c.cv_conv_stride[0];
  auto levels = [&](int64_t n, int* L) {
    L[0] = n >= K0 ? (int)((n - K0) / s0 + 1) : 0;
    for (int i = 1; i < NL; ++i) L[i] = L[i - 1] >= c.cv_conv_kernel[i] ? (L[i - 1] - c.cv_conv_kernel[i]) / c.cv_conv_stride[i] + 1 : 0;
  };
  const int halo = (K0 + s0 - 1) / s0;               // rows of samples past the last frame's window
  auto padded = [&](int L0) { return (L0 + halo + cv_P - 1) / cv_P * cv_P; };
  int64_t mx = 0;
  for (int b = 0; b < B; ++b) {
    REQUIRE(lengths[b] >= 1 && lengths[b] <= ld, VTTS_ERR_INVALID, "wav_lengths must be in [1, wav_ld]");
    int L[8];
    levels(lengths[b], L);
    REQUIRE(L[NL - 1] >= 1, VTTS_ERR_INVALID, "a clip is too short for one ContentVec frame (400 samples at the published shape)");
    REQUIRE(lengths[b] <= (int64_t)1 << 30, VTTS_ERR_INVALID, "clip too long");
    mx = std::max(mx, lengths[b]);
  }
  cvp.maxS = use_buckets ? (int)((mx + 7999) / 8000 * 8000) : (int)mx;
  cvp.maxL.assign(NL, 0);
  levels(cvp.maxS, cvp.maxL.data());
  cvp.MC = (cvp.maxL[0] + CVG_CH - 1) / CVG_CH;
  cvp.nint = (2 * NL + 2) * B;
  std::vector<int>& h = cvp.h;
  h.assign(cvp.nint, 0);
  std::vector<int> frames(B);
  int64_t total0 = 0;                                // layer-0 rows of the batch: every offset (and s0 times it) must fit an int
  for (int b = 0; b < B; ++b) {
    int L[8];
    levels(lengths[b], L);
    total0 += padded(L[0]);
  }
  REQUIRE((total0 + 65535) * s0 + K0 <= (int64_t)INT32_MAX, VTTS_ERR_INVALID, "the batch holds too many samples for one call");
  int off0 = 0;
  for (int b = 0; b < B; ++b) {
    int L[8];
    levels(lengths[b], L);
    int div = 1;
    for (int i = 0; i < NL; ++i) {
      if (i) div *= c.cv_conv_stride[i];
      h[i * B + b] = L[i];
      h[(NL + i) * B + b] = off0 / div;
    }
    h[2 * NL * B + b] = off0 * s0;
    frames[b] = L[NL - 1];
    off0 += padded(L[0]);
  }
  cvp.tot0 = (B == 1 || !use_buckets) ? std::max(off0, use_buckets ? padded(cvp.maxL[0]) : 0) : (off0 + 65535) / 65536 * 65536;
  Staging& s = stg[STG_CONTENTVEC];
  s.begin();
  s.add(d_cvi, cvp.nint);
  s.add(d_cvwav, (size_t)cvp.tot0 * s0 + K0);
  s.commit();
  int* pi = s.host(d_cvi);
  memcpy(pi, h.data(), (size_t)(2 * NL + 1) * B * sizeof(int));
  float* ps = s.host(d_cvwav);
  for (int b = 0; b < B; ++b) {
    const int L0 = h[b];
    const int64_t need = std::min<int64_t>(lengths[b], (int64_t)(L0 - 1) * s0 + K0);
    const float* src = wav + (size_t)b * ld;
    memcpy(ps + h[2 * NL * B + b], src, (size_t)need * sizeof(float));
    double sum = 0.0;                                  // the clip's mean, in one fixed order (layer 0 runs centred on it)
    for (int64_t i = 0; i < lengths[b]; ++i) sum += src[i];
    const float mu = (float)(sum / (double)lengths[b]);
    memcpy(pi + (2 * NL + 1) * B + b, &mu, sizeof(float));
  }
  return frames;
}

// ContentVec of the staged clips (cv_stage): layer 0 + GroupNorm + GELU, layers 1.. (conv_kernel over the strided row view,
// GELU epilogue), LayerNorm + projection, the grouped positional conv (two launches of half the taps each: the tile halo of
// conv_kernel), LayerNorm(x + gelu(pos)), then the post-LN transformer layers.  The last LayerNorm writes frame t of clip b
// to out row out_offs[b] + t (out_offs null: the frame level's own offsets).
void vtts_engine::cv_enqueue(float* out, const int* out_offs, bool fixed) {
  const vtts_config& c = cfg;
  const int NL = c.cv_n_conv, C = c.cv_conv_dim, H = c.cv_hidden, Fh = c.cv_ffn, K0 = c.cv_conv_kernel[0], s0 = c.cv_conv_stride[0];
  // Tensor-core GEMMs without split-K and attention on attn_tc_kernel (Tuning::fixed_tc): a clip's units are then the same
  // alone and in any batch.
  // fixed: every launch in one shape whatever the batch (FFMA convs without split-K, one attention kernel), so that a clip's
  // rows are bit-identical alone and in any batch (SoVITS, whose codes are an argmax of them).
  const Tuning tn = fixed ? (cv_tc ? tune.fixed_ffma().fixed_attention().fixed_tc() : tune.fixed_ffma().fixed_attention())
                          : (cv_tc ? tune.fixed_tc() : tune);
  int* di = ensure(d_cvi, cvp.nint);
  float* dw = ensure(d_cvwav, (size_t)cvp.tot0 * s0 + K0);
  stg[STG_CONTENTVEC].upload();
  auto Ls = [&](int l) -> const int* { return di + l * B; };
  auto Os = [&](int l) -> const int* { return di + (NL + l) * B; };
  const int* woff = di + 2 * NL * B;
  const float* mu = reinterpret_cast<const float*>(di + (2 * NL + 1) * B);
  // the rows of level l; the launch heuristics and the profiler see each clip at the level's bucket
  auto level = [&](int l) { return Rows{Ls(l), Os(l), B, cvp.maxL[l], std::vector<int>(B, cvp.maxL[l]), std::vector<int>(B, cvp.maxL[l]), tn}; };
  const size_t np = (size_t)B * cvp.MC * C;
  float* ps = ensure(d_cvps, np);
  float* pq = ensure(d_cvpq, np);
  float* lv[2] = {ensure(d_cvl[0], (size_t)cvp.tot0 * C), ensure(d_cvl[1], (size_t)cvp.tot0 / c.cv_conv_stride[1] * C)};
  const dim3 gg(cvp.MC, B), gb(CVG_THREADS);
  const size_t gsm = (size_t)((CVG_CH - 1) * s0 + K0) * sizeof(float);
  klaunch(cv_gn_kernel<0>, gg, gb, gsm, (const float*)dw, mu, woff, Ls(0), Os(0), cv_w0, C, K0, s0, ps, pq, cvp.MC, cv_gn_g, cv_gn_b, c.cv_gn_eps, lv[0]);
  CK(cudaGetLastError());
  klaunch(cv_gn_kernel<1>, gg, gb, gsm, (const float*)dw, mu, woff, Ls(0), Os(0), cv_w0, C, K0, s0, ps, pq, cvp.MC, cv_gn_g, cv_gn_b, c.cv_gn_eps, lv[0]);
  CK(cudaGetLastError());
  klaunch(cv_gn_kernel<2>, gg, gb, gsm, (const float*)dw, mu, woff, Ls(0), Os(0), cv_w0, C, K0, s0, ps, pq, cvp.MC, cv_gn_g, cv_gn_b, c.cv_gn_eps, lv[0]);
  CK(cudaGetLastError());
  launches += 3;
  float* x = lv[0];
  for (int i = 1; i < NL; ++i) {
    float* y = lv[i & 1];
    launch_conv({mk(cv_conv[i], x, c.cv_conv_stride[i] * C, 0, y, C, 0, 1, 0)}, 1, level(i));
    gelu_rows(y, C, nullptr, level(i));
    x = y;
  }
  const int* Of = Os(NL - 1);
  const Rows rf = level(NL - 1);
  const size_t Tf = (size_t)cvp.tot0 / cv_P;
  float *X = ensure(d_cvx, Tf * H), *X1 = ensure(d_cvx1, Tf * H), *Y = ensure(d_cvy, Tf * H), *QKV = ensure(d_cvqkv, Tf * 3 * H);
  float *AO = ensure(d_cvao, Tf * std::max(H, C)), *FF = ensure(d_cvff, Tf * Fh);
  // precision modes >= 1: the projection and the transformer's qkv / out / FFN convs on conv_tc_kernel, attention on
  // attn_tc_kernel; every producer of a GEMM operand also writes its split-bf16 planes.  All of
  // them are 1x1, and the attention masks keys past a clip, so no plane row behind a clip is read (no tail zeroing).
  PostLnWs w{X1, X, Y, QKV, AO, FF};
  Planes P512;
  if (cv_tc) {
    P512 = planes(50, (long)Tf, 1, C); w.PX = planes(51, (long)Tf, 1, H); w.PQKV = planes(52, (long)Tf, 1, 3 * H);
    w.PAO = planes(53, (long)Tf, 1, H); w.PX1 = planes(54, (long)Tf, 1, H); w.PFF = planes(55, (long)Tf, 1, Fh);
  }
  ln_rows(x, nullptr, LnW{cv_fp_g, cv_fp_b}, c.cv_ln_eps, AO, Of, C, cv_tc ? &P512 : nullptr, rf);
  if (cv_tc) gemm_rows(P512, cv_tfp, cv_fp, X, nullptr, nullptr, rf);
  else launch_conv({mk(cv_fp, AO, C, 0, X, H, 0, 1, 0)}, 1, rf);
  const int G = c.cv_pos_groups, Cg = H / G, kh = c.cv_pos_k / 2;
  for (int half = 0; half < 2; ++half)
    for (int g0 = 0; g0 < G; g0 += CV_MAXP) {
      std::vector<ConvP> pp;
      for (int g = g0; g < std::min(G, g0 + CV_MAXP); ++g) {
        ConvW W;
        W.w = cv_pos_w + (size_t)(half * G + g) * kh * Cg * Cg;
        W.b = half ? d_cvzero.p : cv_pos_b + (size_t)g * Cg;
        W.Cin = Cg; W.Cout = Cg; W.k = kh; W.ldw = Cg;
        ConvP p = mk(W, X, H, g * Cg, Y, H, g * Cg, 1, half ? c.cv_pos_k / 2 - kh : c.cv_pos_k / 2);
        if (half) { p.res = Y; p.ldr = H; p.roff = g * Cg; }
        pp.push_back(p);
      }
      launch_conv(pp, 1, rf);
    }
  ln_rows(X, Y, LnW{cv_enc_g, cv_enc_b}, c.cv_ln_eps, X1, Of, H, cv_tc ? &w.PX : nullptr, rf);
  if (debug_flags & 1) CK(cudaMemcpyAsync(ensure(d_cvdbg, Tf * H), X1, Tf * H * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  post_ln_layers(cv_enc, cv_tc, H, Fh, c.cv_ln_eps, w, out, out_offs ? out_offs : Of, rf);
}

// SoVITS: ContentVec's tensors (shared binding), then ssl_proj and the codebook scores.
void vtts_engine::bind_sovits() {
  const vtts_config& c = cfg;
  bind_contentvec();
  REQUIRE(has_cv, VTTS_ERR_WEIGHTS, "the weight blob has no HuBERT (cv.*): pack it with weights.pack_sovits");
  const int H = c.cv_hidden;
  sv_K = c.n_vocab;                                // (the codebook's entries: the semantic tokens' vocabulary)
  REQUIRE(sv_K >= 1 && sv_K <= (1 << 16), VTTS_ERR_INVALID, "the codebook (n_vocab) must hold 1 to 65536 entries");
  sv_proj = conv("sv.proj", 2 * H, H, 1);
  sv_score = conv("sv.score", H, sv_K, 1);
}

// Host side of the SoVITS tail: clip b's frames[b] HuBERT rows at row 2 q_b, its frames[b] / 2 pair rows at q_b (an odd last
// frame is dropped, as ssl_proj's stride-2 conv drops it).  feats (vtts_sovits_latent): the caller's rows [B][feats_ld][H],
// staged into those rows; without it ContentVec writes them.
void vtts_engine::sv_stage(const std::vector<int>& frames, int pairs_cap, int maxP, const float* feats, int64_t feats_ld) {
  const int H = cfg.cv_hidden;
  svp.pairs_cap = pairs_cap;
  svp.maxP = maxP;
  svp.frames = frames;
  std::vector<int>& h = svp.h;
  h.assign(3 * B, 0);
  int q = 0;
  for (int b = 0; b < B; ++b) {
    h[b] = 2 * q;
    h[B + b] = frames[b] / 2;
    h[2 * B + b] = q;
    q += (frames[b] + 1) / 2;
  }
  REQUIRE(q <= pairs_cap, VTTS_ERR_STATE, "SoVITS pair rows exceed their buffers");
  Staging& s = stg[STG_SOVITS];
  s.begin();
  s.add(d_svi, 3 * B);
  if (feats) s.add(d_svfeat, (size_t)2 * pairs_cap * H);
  s.commit();
  memcpy(s.host(d_svi), h.data(), h.size() * sizeof(int));
  if (feats) {
    float* pf = s.host(d_svfeat);
    for (int b = 0; b < B; ++b)
      memcpy(pf + (size_t)h[b] * H, feats + (size_t)b * feats_ld * H, (size_t)frames[b] * H * sizeof(float));
  }
}

// The SoVITS tail of the staged clips (sv_stage), after ContentVec of the clips staged by cv_stage when from_wav:
// proj = ssl_proj(pairs), scores = 2 proj.E - |E|^2, codes = the row argmax.  Each output is summed in one order whatever the
// batch (Tuning::fixed_ffma), so a clip's codes are the same alone and in any batch.
void vtts_engine::sv_enqueue(bool from_wav) {
  const int H = cfg.cv_hidden, K = sv_K;
  const size_t P = (size_t)svp.pairs_cap;
  int* di = ensure(d_svi, (size_t)3 * B);
  float* feat = ensure(d_svfeat, 2 * P * H);
  stg[STG_SOVITS].upload();
  if (from_wav) cv_enqueue(feat, di, true);
  float* proj = ensure(d_svproj, P * H);
  float* score = ensure(d_svscore, P * K);
  int* codes = ensure(d_svcodes, P);
  std::vector<int> real(B);
  for (int b = 0; b < B; ++b) real[b] = svp.h[B + b];
  const Rows r{di + B, di + 2 * B, B, svp.maxP, std::vector<int>(B, svp.maxP), real, tune.fixed_ffma()};
  launch_conv({mk(sv_proj, feat, 2 * H, 0, proj, H, 0, 1, 0)}, 1, r);
  launch_conv({mk(sv_score, proj, H, 0, score, K, 0, 1, 0)}, 1, r);
  klaunch(sv_argmax_kernel, dim3((std::max(svp.maxP, 1) + SVA_WARPS - 1) / SVA_WARPS, B), dim3(32 * SVA_WARPS), (size_t)0,
          (const float*)score, K, (const int*)(di + B), (const int*)(di + 2 * B), codes);
  CK(cudaGetLastError());
  ++launches;
}

// LayerNorm of the rows r (cv_ln_kernel): out = LN(a + gelu(y)) (y null: LN(a)), rows read at r.offs, written at out_offs.
void vtts_engine::ln_rows(const float* a, const float* y, const LnW& w, float eps, float* out, const int* out_offs, int C,
                          const Planes* pl, const Rows& r) {
  klaunch(cv_ln_kernel, dim3((r.maxLen + CVL_WARPS - 1) / CVL_WARPS, r.n), dim3(32 * CVL_WARPS), (size_t)0, a, y, w.g, w.b, eps, out,
          r.lens, r.offs, out_offs, C, pl ? pl->hi : (__nv_bfloat16*)nullptr, pl ? pl->lo : (__nv_bfloat16*)nullptr);
  CK(cudaGetLastError());
  ++launches;
}

// GELU of the rows r (cv_gelu_kernel): in place, or into the planes pl.
void vtts_engine::gelu_rows(float* y, int C, const Planes* pl, const Rows& r) {
  klaunch(cv_gelu_kernel, dim3(r.maxLen, r.n), dim3(256), (size_t)0, y, C, r.lens, r.offs, pl ? pl->hi : (__nv_bfloat16*)nullptr,
          pl ? pl->lo : (__nv_bfloat16*)nullptr);
  CK(cudaGetLastError());
  ++launches;
}

// One 1x1 conv of the rows r on the tensor cores: y = in W^T + bias (+ res), and the planes of y when out is given.
void vtts_engine::gemm_rows(const Planes& in, const TcW& w, const ConvW& cw, float* y, const float* res, const Planes* out, const Rows& r) {
  TcSpec s;
  s.in = in; s.w = w; s.bias = cw.b; s.Cin = cw.Cin; s.Cout = cw.Cout;
  s.y = y; s.ldy = cw.Cout; s.res = res; s.ldr = res ? cw.Cout : 0; s.epi = 0;
  if (out) s.out = *out;
  launch_tc({s}, 1, r);
}

// The post-LN transformer layers of ContentVec (HubertEncoderLayer), BERT (BertLayer) and GPT-SoVITS's text prefill
// (TransformerEncoderLayer; relu): x = LN(x + o(attention(qkv(x)))), x = LN(x + ffn2(act(ffn1(x)))), act GELU or ReLU, with no relative positions (relk / relv of every layer point at zeros).  The input rows are
// w.xa (on_tc: and their planes w.PX); the last LayerNorm writes row t of sequence b to out row out_offs[b] + t.  on_tc: the
// convs on conv_tc_kernel and the attention on attn_tc_kernel where r.tune takes it, else everything on the FFMA pipe.
// after_qkv (or null) is called with the layer index right behind each layer's qkv GEMM, whose rows w.QKV then holds.
// prefix (or null): [B][4] ints whose first is the text length T of each sequence; the attention then runs under
// GPT-SoVITS's prefix mask (t2s_prefix_attn_kernel: row t sees key k iff k < T or k <= t) on the fp32 qkv rows.
void vtts_engine::post_ln_layers(const std::vector<EncLayerW>& layers, bool on_tc, int H, int Fh, float eps, PostLnWs w,
                                 float* out, const int* out_offs, const Rows& r, bool relu, const std::function<void(int)>* after_qkv,
                                 const int* prefix) {
  float *xa = w.xa, *xb = w.xb;
  auto prefix_attn = [&](const EncLayerW& Lw, const Planes* pl) {
    const int dk = H / Lw.heads;
    klaunch(t2s_prefix_attn_kernel, dim3(r.maxLen, Lw.heads, r.n), dim3(32), (size_t)0, (const float*)w.QKV, H, dk,
            (float)std::sqrt(1.0 / dk), w.AO, r.lens, r.offs, prefix, pl ? pl->hi : (__nv_bfloat16*)nullptr,
            pl ? pl->lo : (__nv_bfloat16*)nullptr);
    CK(cudaGetLastError());
    ++launches;
  };
  auto act = [&](const Planes* pl) {
    if (!relu) { gelu_rows(w.FF, Fh, pl, r); return; }
    klaunch(t2s_relu_kernel, dim3(r.maxLen, r.n), dim3(256), (size_t)0, w.FF, Fh, r.lens, r.offs, pl ? pl->hi : (__nv_bfloat16*)nullptr,
            pl ? pl->lo : (__nv_bfloat16*)nullptr);
    CK(cudaGetLastError());
    ++launches;
  };
  for (size_t l = 0; l < layers.size() && on_tc; ++l) {
    const EncLayerW& Lw = layers[l];
    gemm_rows(w.PX, Lw.t_qkv, Lw.qkv, w.QKV, nullptr, &w.PQKV, r);
    if (after_qkv) (*after_qkv)((int)l);
    if (prefix) prefix_attn(Lw, &w.PAO);
    else if (attn_use_tc(Lw, H, r)) launch_attn_tc(w.PQKV, w.AO, &w.PAO, Lw, H, r);
    else launch_attn(w.QKV, w.AO, Lw, H, &w.PAO, r);
    gemm_rows(w.PAO, Lw.t_o, Lw.o, w.Y, xa, nullptr, r);
    ln_rows(w.Y, nullptr, Lw.ln1, eps, xb, r.offs, H, &w.PX1, r);
    gemm_rows(w.PX1, Lw.t_ffn1, Lw.ffn1, w.FF, nullptr, nullptr, r);
    act(&w.PFF);
    gemm_rows(w.PFF, Lw.t_ffn2, Lw.ffn2, w.Y, xb, nullptr, r);
    if (l + 1 == layers.size()) ln_rows(w.Y, nullptr, Lw.ln2, eps, out, out_offs, H, nullptr, r);
    else ln_rows(w.Y, nullptr, Lw.ln2, eps, xa, r.offs, H, &w.PX, r);
  }
  for (size_t l = 0; l < layers.size() && !on_tc; ++l) {
    const EncLayerW& Lw = layers[l];
    launch_conv({mk(Lw.qkv, xa, H, 0, w.QKV, 3 * H, 0, 1, 0)}, 1, r);
    if (after_qkv) (*after_qkv)((int)l);
    if (prefix) prefix_attn(Lw, nullptr);
    else launch_attn(w.QKV, w.AO, Lw, H, nullptr, r);
    ConvP po = mk(Lw.o, w.AO, H, 0, w.Y, H, 0, 1, 0);
    po.res = xa; po.ldr = H;
    launch_conv({po}, 1, r);
    ln_rows(w.Y, nullptr, Lw.ln1, eps, xb, r.offs, H, nullptr, r);
    launch_conv({mk(Lw.ffn1, xb, H, 0, w.FF, Fh, 0, 1, 0)}, 1, r);
    act(nullptr);
    ConvP p2 = mk(Lw.ffn2, w.FF, Fh, 0, w.Y, H, 0, 1, 0);
    p2.res = xb; p2.ldr = H;
    launch_conv({p2}, 1, r);
    if (l + 1 == layers.size()) ln_rows(w.Y, nullptr, Lw.ln2, eps, out, out_offs, H, nullptr, r);
    else ln_rows(w.Y, nullptr, Lw.ln2, eps, xa, r.offs, H, nullptr, r);
  }
}

// ---------------------------------------------------------------------------------------------------
// BERT (transformers' BertModel as training/stabletts/matcha/onnx/bert-export.py exports it: hidden_states[-3], i.e. the output
// of the last layer the blob holds; bert.cuh)
// ---------------------------------------------------------------------------------------------------
void vtts_engine::bind_bert() {
  const vtts_config& c = cfg;
  has_bert = tensors.count("bt.emb.word") > 0;
  if (!has_bert) return;
  const int H = c.cv_hidden, Fh = c.cv_ffn, nh = c.cv_heads;
  REQUIRE(c.cv_layers >= 1 && nh >= 1 && H % nh == 0 && (H / nh) % 32 == 0 && H / nh <= 128 && H % CV_CK == 0 && H <= 32 * CVL_MAXV &&
              Fh >= CV_CK && Fh % CV_CK == 0,
          VTTS_ERR_INVALID, "unsupported BERT shape (at least one layer, head width a multiple of 32 up to 128, width a multiple of 16 "
          "up to 1024, FFN a multiple of 16)");
  REQUIRE(c.cv_ln_eps > 0.f, VTTS_ERR_INVALID, "BERT needs a positive LayerNorm eps");
  // the tables' rows are the blob's: vocabulary, positions (the longest sentence) and token types
  auto rows = [&](const char* name) {
    const size_t n = tensor(name).n;
    REQUIRE(n >= (size_t)H && n % H == 0 && n / H <= (size_t)INT32_MAX, VTTS_ERR_WEIGHTS, std::string("bad BERT table ") + name);
    return (int)(n / H);
  };
  bt_vocab = rows("bt.emb.word");
  bt_max_pos = rows("bt.emb.pos");
  bt_tc = c.precision >= 1 && c.precision <= 3;
  if (bt_tc) {
    REQUIRE(H % TC_BK == 0 && Fh % TC_BK == 0, VTTS_ERR_INVALID, "BERT on the tensor cores needs widths in multiples of 64");
    REQUIRE(tensors.count("bt.l0.qkv.th") > 0, VTTS_ERR_WEIGHTS, "the blob lacks BERT's tensor-core weights");
  }
  bt_word = vec("bt.emb.word", (size_t)bt_vocab * H);
  bt_pos = vec("bt.emb.pos", (size_t)bt_max_pos * H);
  bt_type = vec("bt.emb.type", (size_t)rows("bt.emb.type") * H);
  bt_ln = ln("bt.emb.ln", H);
  // zeros: the relative tables of the attention (fp32, and the [16][128] bf16 tiles of the tensor-core attention).  BERT has
  // absolute positions only; the attention kernels always add a relative term, which these zeros make vanish exactly.  A
  // StableTTS engine leaves window_size 0 (make_c_config does not set it), so that term is one offset per query row.
  const size_t nz = std::max<size_t>({(size_t)H, (size_t)(2 * c.window_size + 1) * (H / nh), (size_t)ATC_RELP * 128});
  float* zero = ensure(d_btzero, nz);
  CK(cudaMemsetAsync(zero, 0, d_btzero.cap * sizeof(float), stream));
  bt_enc.clear();
  for (int l = 0; l < c.cv_layers; ++l) {
    const std::string p = "bt.l" + std::to_string(l);
    EncLayerW L;
    L.heads = nh;
    L.qkv = conv(p + ".qkv", H, 3 * H, 1);
    L.o = conv(p + ".o", H, H, 1);
    L.ln1 = ln(p + ".ln1", H);
    L.ffn1 = conv(p + ".ffn1", H, Fh, 1);
    L.ffn2 = conv(p + ".ffn2", Fh, H, 1);
    L.ln2 = ln(p + ".ln2", H);
    L.relk = L.relv = zero;
    if (bt_tc) {
      L.t_qkv = tcw(p + ".qkv", H, 3 * H, 1);
      L.t_o = tcw(p + ".o", H, H, 1);
      L.t_ffn1 = tcw(p + ".ffn1", H, Fh, 1);
      L.t_ffn2 = tcw(p + ".ffn2", Fh, H, 1);
      const __nv_bfloat16* zb = reinterpret_cast<const __nv_bfloat16*>(zero);
      L.rk_hi = L.rk_lo = L.rv_hi = L.rv_lo = zb;
    }
    bt_enc.push_back(L);
  }
}

// Host side of a BERT call: validates the word pieces and packs the sentences' rows back to back (each starting at a multiple
// of 8), then stages [len B][off B][ids] in pinned memory.  The longest sentence and the row total are bucketed (32 rows; 1024
// rows for batches), so a captured graph serves every call of the bucket.
void vtts_engine::bt_stage(const int64_t* ids, const int64_t* lengths, int64_t ld) {
  const vtts_config& c = cfg;
  btp.len.assign(B, 0);
  btp.off.assign(B, 0);
  int mx = 0, tot = 0;
  for (int b = 0; b < B; ++b) {
    REQUIRE(lengths[b] >= 1 && lengths[b] <= ld, VTTS_ERR_INVALID, "lengths must be in [1, ids_ld]");
    REQUIRE(lengths[b] <= bt_max_pos, VTTS_ERR_INVALID, "a sentence is longer than BERT's position table (max_position_embeddings)");
    for (int64_t t = 0; t < lengths[b]; ++t) {
      const int64_t v = ids[(size_t)b * ld + t];
      REQUIRE(v >= 0 && v < bt_vocab, VTTS_ERR_INVALID, "a word-piece id is outside BERT's vocabulary");
    }
    btp.len[b] = (int)lengths[b];
    btp.off[b] = tot;
    tot += (btp.len[b] + 7) / 8 * 8;
    REQUIRE(tot <= (1 << 24), VTTS_ERR_INVALID, "the batch holds too many word pieces for one call");
    mx = std::max(mx, btp.len[b]);
  }
  btp.maxL = use_buckets ? (mx + 31) / 32 * 32 : mx;
  btp.tot = !use_buckets ? tot : B == 1 ? btp.maxL : (tot + 1023) / 1024 * 1024;
  Staging& s = stg[STG_BERT];
  s.begin();
  s.add(d_bti, 2 * (size_t)B + btp.tot);
  s.commit();
  int* pin = s.host(d_bti);
  memcpy(pin, btp.len.data(), B * sizeof(int));
  memcpy(pin + B, btp.off.data(), B * sizeof(int));
  std::fill(pin + 2 * B, pin + 2 * B + btp.tot, 0);
  for (int b = 0; b < B; ++b)
    for (int t = 0; t < btp.len[b]; ++t) pin[2 * B + btp.off[b] + t] = (int)ids[(size_t)b * ld + t];
}

// BERT of the staged sentences (bt_stage): the embeddings, then the post-LN layers; the last LayerNorm writes the packed rows
// to out.  Every launch has one shape whatever the batch (Tuning::fixed_ffma and fixed_attention in mode 0, fixed_tc in modes
// >= 1), so a sentence's rows are the same alone and in any batch.
void vtts_engine::bt_enqueue(float* out) {
  const vtts_config& c = cfg;
  const int H = c.cv_hidden, Fh = c.cv_ffn;
  const Tuning tn = bt_tc ? tune.fixed_tc() : tune.fixed_ffma().fixed_attention();
  const size_t T = btp.tot, nint = 2 * (size_t)B + T;
  int* di = ensure(d_bti, nint);
  stg[STG_BERT].upload();
  const Rows r{di, di + B, B, btp.maxL, std::vector<int>(B, btp.maxL), btp.len, tn};
  PostLnWs w{ensure(d_btx, T * H), ensure(d_btx1, T * H), ensure(d_bty, T * H), ensure(d_btqkv, T * 3 * H), ensure(d_btao, T * H),
             ensure(d_btff, T * Fh)};
  if (bt_tc) {
    w.PX = planes(51, (long)T, 1, H); w.PQKV = planes(52, (long)T, 1, 3 * H);
    w.PAO = planes(53, (long)T, 1, H); w.PX1 = planes(54, (long)T, 1, H); w.PFF = planes(55, (long)T, 1, Fh);
  }
  klaunch(bert_embed_kernel, dim3((btp.maxL + CVL_WARPS - 1) / CVL_WARPS, B), dim3(32 * CVL_WARPS), (size_t)0, (const int*)(di + 2 * B),
          bt_word, bt_pos, bt_type, bt_ln.g, bt_ln.b, c.cv_ln_eps, w.xa, r.lens, r.offs, H, bt_tc ? w.PX.hi : (__nv_bfloat16*)nullptr,
          bt_tc ? w.PX.lo : (__nv_bfloat16*)nullptr);
  CK(cudaGetLastError());
  ++launches;
  post_ln_layers(bt_enc, bt_tc, H, Fh, c.cv_ln_eps, w, out, r.offs, r);
}

// ---------------------------------------------------------------------------------------------------
// GPT-SoVITS text-to-semantic decoder (Text2SemanticDecoder, training/gpt-sovits/ar/models/t2s_model.py:324-448; t2s.cuh)
// ---------------------------------------------------------------------------------------------------
void vtts_engine::bind_t2s() {
  const vtts_config& c = cfg;
  const int H = c.cv_hidden, F = c.cv_ffn, nh = c.cv_heads;
  REQUIRE(c.cv_layers >= 1 && nh >= 1 && H % nh == 0 && (H / nh) % 32 == 0 && H / nh <= 128 && H % CV_CK == 0 && H <= 32 * CVL_MAXV &&
              F >= CV_CK && F % T2S_WARPS == 0 && F <= T2S_MAX_V,
          VTTS_ERR_INVALID, "unsupported text-to-semantic shape (at least one layer, head width a multiple of 32 up to 128, width a "
          "multiple of 32 up to 1024, FFN a multiple of 32 up to 4096)");
  REQUIRE(c.cv_ln_eps > 0.f, VTTS_ERR_INVALID, "the text-to-semantic decoder needs a positive LayerNorm eps");
  auto rows = [&](const char* name) {
    const size_t n = tensor(name).n;
    REQUIRE(n >= (size_t)H && n % H == 0 && n / H <= (size_t)INT32_MAX, VTTS_ERR_WEIGHTS, std::string("bad text-to-semantic table ") + name);
    return (int)(n / H);
  };
  t2s_text_vocab = rows("t2s.temb");
  t2s_vocab = rows("t2s.aemb");
  t2s_npos = rows("t2s.pe");
  REQUIRE(t2s_vocab >= 2 && t2s_vocab <= T2S_MAX_V, VTTS_ERR_INVALID, "the semantic vocabulary (EOS included) must have 2 to 4096 entries");
  t2s_temb = vec("t2s.temb", (size_t)t2s_text_vocab * H);
  t2s_aemb = vec("t2s.aemb", (size_t)t2s_vocab * H);
  t2s_pe = vec("t2s.pe", (size_t)t2s_npos * H);
  CK(cudaMemcpy(t2s_alpha, vec("t2s.alpha", 2), 2 * sizeof(float), cudaMemcpyDeviceToHost));
  t2s_bp = conv("t2s.bert_proj", T2S_BERT, H, 1);
  t2s_pred = conv("t2s.pred", H, t2s_vocab, 1);
  t2s_tc = c.precision >= 1 && c.precision <= 3;
  if (t2s_tc) {
    REQUIRE(H % TC_BK == 0 && F % TC_BK == 0, VTTS_ERR_INVALID, "the text prefill on the tensor cores needs widths in multiples of 64");
    REQUIRE(tensors.count("t2s.l0.qkv.th") > 0, VTTS_ERR_WEIGHTS, "the blob lacks the text prefill's tensor-core weights");
  }
  // zeros for the attention's relative terms, which post_ln_layers' kernels always add (as bind_bert)
  const size_t nz = std::max<size_t>({(size_t)H, (size_t)(2 * c.window_size + 1) * (H / nh), (size_t)ATC_RELP * 128});
  float* zero = ensure(d_t2s_zero, nz);
  CK(cudaMemsetAsync(zero, 0, d_t2s_zero.cap * sizeof(float), stream));
  t2s_enc.clear();
  for (int l = 0; l < c.cv_layers; ++l) {
    const std::string p = "t2s.l" + std::to_string(l);
    EncLayerW L;
    L.heads = nh;
    L.qkv = conv(p + ".qkv", H, 3 * H, 1);
    L.o = conv(p + ".o", H, H, 1);
    L.ln1 = ln(p + ".ln1", H);
    L.ffn1 = conv(p + ".ffn1", H, F, 1);
    L.ffn2 = conv(p + ".ffn2", F, H, 1);
    L.ln2 = ln(p + ".ln2", H);
    L.relk = L.relv = zero;
    if (t2s_tc) {
      L.t_qkv = tcw(p + ".qkv", H, 3 * H, 1);
      L.t_o = tcw(p + ".o", H, H, 1);
      L.t_ffn1 = tcw(p + ".ffn1", H, F, 1);
      L.t_ffn2 = tcw(p + ".ffn2", F, H, 1);
      const __nv_bfloat16* zb = reinterpret_cast<const __nv_bfloat16*>(zero);
      L.rk_hi = L.rk_lo = L.rv_hi = L.rv_lo = zb;
    }
    t2s_enc.push_back(L);
  }
  CK(cudaFuncSetAttribute(t2s_ffn2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T2S_GEMV_SMEM(F)));
}

// ---------------------------------------------------------------------------------------------------
// StableTTS flow-matching decoder (flow_matching.py:33-100,182-194; decoder.py:103-138; diffusion_transformer.py:98-116)
// ---------------------------------------------------------------------------------------------------
void vtts_engine::bind_stabletts() {
  const vtts_config& c = cfg;
  const int NC = c.st_noise, MC = c.st_cond, H = c.st_hidden, F = c.st_filter, NL = c.st_layers, G = c.st_spk_dim, k = c.st_kernel;
  REQUIRE(NL >= 2 && NL % 2 == 0 && NL <= 8, VTTS_ERR_INVALID, "unsupported StableTTS decoder: the U-Net long skips need an even number of blocks (2..8)");
  REQUIRE(c.st_heads >= 1 && H % c.st_heads == 0 && (H / c.st_heads) % 32 == 0 && H / c.st_heads <= 128 && (H / c.st_heads) % 4 == 0,
          VTTS_ERR_INVALID, "unsupported StableTTS decoder: the attention kernels take head widths 32, 64, 96 and 128");
  REQUIRE(H % CV_CK == 0 && H <= 32 * DIT_LN_MAXV && F % CV_CK == 0 && F <= DIT_MAXC && MC % CV_CK == 0 && (NC + H) % CV_CK == 0 && NC % 4 == 0 &&
              G >= 1 && G <= DIT_MAXC && k % 2 == 1 && k >= 1 && k <= 15 && c.st_n_spks >= 1,
          VTTS_ERR_INVALID, "unsupported StableTTS decoder (widths in multiples of 16, hidden up to 512, filter up to 1024, odd kernel)");
  st_cp[0] = conv("st.cp0", MC, F, k);
  st_cp[1] = conv("st.cp1", F, F, k);
  st_cp[2] = conv("st.cp2", F, H, k);
  st_in = conv("st.in", NC + H, H, 1);
  st_final = conv("st.final", H, NC, 1);
  st_tw1 = vec("st.time.w1", (size_t)F * H); st_tb1 = vec("st.time.b1", F);
  st_tw2 = vec("st.time.w2", (size_t)H * F); st_tb2 = vec("st.time.b2", H);
  st_fw = vec("st.film.w", (size_t)NL * 2 * H * H); st_fb = vec("st.film.b", (size_t)NL * 2 * H);
  st_aw1 = vec("st.ada.w1", (size_t)NL * H * G); st_ab1 = vec("st.ada.b1", (size_t)NL * H);
  st_aw2 = vec("st.ada.w2", (size_t)NL * 6 * H * H); st_ab2 = vec("st.ada.b2", (size_t)NL * 6 * H);
  st_emb = vec("st.spk_emb", (size_t)c.st_n_spks * G);
  st_fake_spk = vec("st.fake_spk", G);
  st_fake_content = vec("st.fake_content", MC);
  st_mel_mean = vec("st.mel_mean", 1);
  st_mel_std = vec("st.mel_std", 1);
  float* zero = ensure(d_stzero, (size_t)H);       // the attention's relative tables: no window, both terms exact zeros
  CK(cudaMemsetAsync(zero, 0, d_stzero.cap * sizeof(float), stream));
  st_blk.clear();
  st_lsc.clear();
  for (int l = 0; l < NL; ++l) {
    const std::string p = "st.l" + std::to_string(l);
    EncLayerW L;
    L.heads = c.st_heads;
    L.qkv = conv(p + ".qkv", H, 3 * H, 1);
    L.o = conv(p + ".o", H, H, 1);
    L.ffn1 = conv(p + ".ffn1", H, F, k);
    L.ffn2 = conv(p + ".ffn2", F, H, k);
    L.relk = L.relv = zero;
    st_blk.push_back(L);
    if (l >= NL / 2) st_lsc.push_back(conv("st.lsc" + std::to_string(l - NL / 2), 2 * H, H, k));
  }
  // precision mode 2: each conv's pipe (st_tc_fits), its split-bf16 weights (weights.pack_stabletts*(..., precision=2)), and
  // the attention on attn_tc_kernel with zero relative tiles, as BERT runs it (bind_bert)
  stp_tc = StPipe{};
  st_tlsc.clear();
  if (c.precision == 2) {
    StPipe& p = stp_tc;
    p.on = true;
    p.cp[0] = st_tc_fits(MC, F); p.cp[1] = st_tc_fits(F, F); p.cp[2] = st_tc_fits(F, H);
    p.qkv = st_tc_fits(H, 3 * H); p.o = st_tc_fits(H, H); p.ffn1 = st_tc_fits(H, F); p.ffn2 = st_tc_fits(F, H); p.lsc = st_tc_fits(2 * H, H);
    const char* first = p.qkv ? "st.l0.qkv" : p.o ? "st.l0.o" : p.ffn1 ? "st.l0.ffn1" : p.ffn2 ? "st.l0.ffn2" : p.lsc ? "st.lsc0"
                      : p.cp[0] ? "st.cp0" : p.cp[1] ? "st.cp1" : p.cp[2] ? "st.cp2" : nullptr;
    REQUIRE(!first || tensors.count(std::string(first) + ".th"), VTTS_ERR_WEIGHTS,
            "the blob lacks the StableTTS decoder's tensor-core weights (pack it with precision=2)");
    for (int i = 0; i < 3; ++i)
      if (p.cp[i]) st_tcp[i] = tcw("st.cp" + std::to_string(i), st_cp[i].Cin, st_cp[i].Cout, k);
    for (int j = 0; j < NL / 2 && p.lsc; ++j) st_tlsc.push_back(tcw("st.lsc" + std::to_string(j), 2 * H, H, k));
    const int dk = H / c.st_heads;
    p.attn = dk % 32 == 0 && dk <= 128 && c.window_size == 0;
    float* z = ensure(d_stzero, std::max<size_t>((size_t)H, (size_t)ATC_RELP * 128));     // (the [16][128] bf16 tiles as well)
    CK(cudaMemsetAsync(z, 0, d_stzero.cap * sizeof(float), stream));
    zero = z;                                        // (the text encoder's tables below point here too)
    const __nv_bfloat16* zb = reinterpret_cast<const __nv_bfloat16*>(z);
    for (int l = 0; l < NL; ++l) {
      EncLayerW& L = st_blk[l];
      const std::string q = "st.l" + std::to_string(l);
      L.relk = L.relv = z;
      if (p.qkv) L.t_qkv = tcw(q + ".qkv", H, 3 * H, 1);
      if (p.o) L.t_o = tcw(q + ".o", H, H, 1);
      if (p.ffn1) L.t_ffn1 = tcw(q + ".ffn1", H, F, k);
      if (p.ffn2) L.t_ffn2 = tcw(q + ".ffn2", F, H, k);
      if (p.attn) L.rk_hi = L.rk_lo = L.rv_hi = L.rv_lo = zb;
    }
  }
  // the vocoder, when the blob carries it (weights.pack_hifigan): described by the decoder fields of the config
  has_voc = tensors.count("dec.pre.w") > 0;
  if (has_voc) {
    REQUIRE(c.decoder_type == 1, VTTS_ERR_INVALID, "unsupported vocoder: only the HiFi-GAN Generator (decoder_type 1) is built");
    REQUIRE(c.inter_channels == NC, VTTS_ERR_INVALID, "unsupported vocoder: conv_pre's input (inter_channels) must equal st_noise");
    REQUIRE(c.n_upsamples >= 1 && c.n_upsamples <= 8 && c.n_resblock_kernels >= 1 && c.n_resblock_dilations >= 1 &&
                c.n_resblock_dilations <= 8 && (c.upsample_initial_channel >> c.n_upsamples) >= CV_CK &&
                (c.upsample_initial_channel >> c.n_upsamples) << c.n_upsamples == c.upsample_initial_channel,
            VTTS_ERR_INVALID, "unsupported vocoder: 1..8 upsampling stages halving upsample_initial_channel to a multiple of 16");
    REQUIRE(c.n_resblock_kernels <= 3, VTTS_ERR_INVALID, "unsupported vocoder: at most 3 resblocks per stage");
    for (int i = 0; i < c.n_upsamples; ++i)
      REQUIRE(c.upsample_rates[i] >= 1 && c.upsample_kernel_sizes[i] >= c.upsample_rates[i] && (c.upsample_kernel_sizes[i] - c.upsample_rates[i]) % 2 == 0,
              VTTS_ERR_INVALID, "unsupported vocoder: every ConvTranspose1d needs kernel - rate even and >= 0 (padding (k - u) / 2 gives u T rows)");
    bind_decoder();       // (also refuses a receptive field wider than the conv tile)
  }
  // the text encoder, when the blob carries it (weights.pack_stabletts); a decoder-only blob serves vtts_cfm_decode alone
  st_text = c.st_enc_layers > 0;
  if (!st_text) return;
  const int He = c.st_enc_hidden, Fe = c.st_enc_filter, NE = c.st_enc_layers, ke = c.st_enc_kernel;
  REQUIRE(tensors.count("st.enc.emb"), VTTS_ERR_WEIGHTS, "the config describes a StableTTS text encoder the weight blob does not carry");
  REQUIRE(c.st_streams >= 1 && c.st_streams <= 8 && c.st_emb_dim >= 1 && c.st_punc_dim >= 1 && c.st_bert_proj >= 1 && c.st_n_vocab >= 1 &&
              c.st_emb_dim + (c.st_streams - 1) * c.st_punc_dim + c.st_bert_proj == MC && He == MC,
          VTTS_ERR_INVALID, "unsupported StableTTS text encoder: the embeddings and bert_proj must concatenate to cond_channels, the stacks' width");
  REQUIRE(c.st_bert_dim >= 1 && c.st_bert_dim <= STT_MAXBERT && c.st_dur_channels >= 1 && c.st_dur_channels <= 1024, VTTS_ERR_INVALID,
          "unsupported StableTTS text encoder: BERT rows up to 1024 wide, up to 1024 duration channels");
  REQUIRE(NE >= 1 && NE <= 8 && c.st_enc_heads >= 1 && He % c.st_enc_heads == 0 && (He / c.st_enc_heads) % 32 == 0 && He / c.st_enc_heads <= 128 &&
              He % CV_CK == 0 && He <= 32 * DIT_LN_MAXV && Fe % CV_CK == 0 && Fe <= DIT_MAXC && ke % 2 == 1 && ke >= 1 && ke <= 15,
          VTTS_ERR_INVALID, "unsupported StableTTS text encoder (head widths 32..128, hidden up to 512, filter up to 1024, odd kernel)");
  st_tok_emb = vec("st.enc.emb", (size_t)c.st_n_vocab * c.st_emb_dim);
  st_punc_emb = vec("st.enc.punc", (size_t)c.st_n_vocab * c.st_punc_dim);
  st_bert_w = vec("st.enc.bert.w", (size_t)c.st_bert_proj * c.st_bert_dim);
  st_bert_b = vec("st.enc.bert.b", c.st_bert_proj);
  // the mel encoder feeds only the prior (encoder_outputs); an exported graph (matcha/onnx/export.py) does not output it and
  // so does not carry its weights
  st_prior = tensors.count("st.enc.mel.proj.w") > 0;
  for (int e = st_prior ? 0 : 1; e < 2; ++e) {
    const std::string p = e == 0 ? "st.enc.mel" : "st.enc.dp";
    StEncW& W = st_enc[e];
    W.blk.clear();
    for (int l = 0; l < NE; ++l) {
      const std::string q = p + ".l" + std::to_string(l);
      EncLayerW L;
      L.heads = c.st_enc_heads;
      L.qkv = conv(q + ".qkv", He, 3 * He, 1);
      L.o = conv(q + ".o", He, He, 1);
      L.ffn1 = conv(q + ".ffn1", He, Fe, ke);
      L.ffn2 = conv(q + ".ffn2", Fe, He, ke);
      L.relk = L.relv = zero;
      W.blk.push_back(L);
    }
    W.proj = conv(p + ".proj", He, e == 0 ? NC : c.st_dur_channels, 1);
    W.aw1 = vec(p + ".ada.w1", (size_t)NE * He * G); W.ab1 = vec(p + ".ada.b1", (size_t)NE * He);
    W.aw2 = vec(p + ".ada.w2", (size_t)NE * 6 * He * He); W.ab2 = vec(p + ".ada.b2", (size_t)NE * 6 * He);
    W.spk = e == 0 ? st_emb : vec("st.dur_spk_emb", (size_t)c.st_n_spks * G);
  }
}

// modulated LayerNorm -> qkv 1x1 -> rotary -> attention (zero relative tables) -> out 1x1 -> gated residual + modulated
// LayerNorm -> conv -> SiLU -> conv -> gated residual; x rows at xin (pitch ldi) -> xout (pitch ldo).  film: the FiLM rows
// DitWrapper applies first (decoder.py:15-18), or null for the text encoder's plain blocks.
void vtts_engine::st_block(const StBlk& k, const EncLayerW& L, int l, const float* film, const float* xin, int ldi, float* xout, int ldo, bool tap,
                           const Rows& r) {
  const int H = k.H, F = k.F, dk = H / k.heads;
  const size_t T = (size_t)stp.Ttot;
  const dim3 gs(r.maxLen, r.n), gn((r.maxLen + DIT_LN_WARPS - 1) / DIT_LN_WARPS, r.n);
  const float* ada = k.ada + (size_t)l * 6 * H;
  auto norm = [&](const float* a, int lda, const float* fl, const float* y, int gate, int shift, int scale) {
    klaunch(dit_norm_kernel, gn, dim3(32 * DIT_LN_WARPS), (size_t)0, a, lda, fl, y, ada, k.ald, gate * H, shift * H, scale * H, 1e-5f, k.Hb, k.N,
            r.lens, r.offs, H);
    CK(cudaGetLastError());
    ++launches;
  };
  auto cv = [&](const ConvW& W, const float* x, int ldx, float* y, int ldy) {
    launch_conv({mk(W, x, ldx, 0, y, ldy, 0, 1, (W.k - 1) / 2)}, 1, r);
  };
  norm(xin, ldi, film, nullptr, 2, 0, 1);
  if (tap) CK(cudaMemcpyAsync(ensure(d_stdbg_n, T * H), k.N, T * H * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  cv(L.qkv, k.N, H, k.QKV, 3 * H);
  klaunch(dit_rope_kernel, gs, dim3(128), (size_t)0, k.QKV, k.rope, k.heads, dk, k.rd, r.lens, r.offs);
  CK(cudaGetLastError());
  ++launches;
  if (tap) CK(cudaMemcpyAsync(ensure(d_stdbg_qkv, T * 3 * H), k.QKV, T * 3 * H * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  launch_attn(k.QKV, k.AO, L, H, nullptr, r);
  cv(L.o, k.AO, H, k.Y, H);
  norm(k.Hb, H, nullptr, k.Y, 2, 3, 4);
  cv(L.ffn1, k.N, H, k.FF, F);
  klaunch(dit_silu_kernel, gs, dim3(256), (size_t)0, k.FF, F, r.lens, r.offs);
  CK(cudaGetLastError());
  ++launches;
  cv(L.ffn2, k.FF, F, k.Y, H);
  klaunch(dit_gate_kernel, gs, dim3(128), (size_t)0, (const float*)k.Hb, (const float*)k.Y, ada, k.ald, 5 * H, xout, ldo, r.lens, r.offs, H);
  CK(cudaGetLastError());
  ++launches;
}

// st_block with the convs stp_tc takes on conv_tc_kernel and the attention on attn_tc_kernel (precision mode 2, the mel phase
// only).  Every producer still writes its fp32 rows; those that feed a tensor-core operand also write its planes (stpl).
void vtts_engine::st_block_tc(const StBlk& k, const EncLayerW& L, int l, const float* film, const float* xin, int ldi, float* xout, int ldo,
                              const Planes* xout_pl, bool tap, const Rows& r) {
  const StPipe& p = stp_tc;
  const StPl& pl = stpl;
  const int H = k.H, F = k.F, dk = H / k.heads;
  const size_t T = (size_t)stp.Ttot;
  const dim3 gs(r.maxLen, r.n), gn((r.maxLen + DIT_LN_WARPS - 1) / DIT_LN_WARPS, r.n);
  const float* ada = k.ada + (size_t)l * 6 * H;
  const bool attn_tc = p.attn && attn_use_tc(L, H, r);
  auto norm = [&](const float* a, int lda, const float* fl, const float* y, int gate, int shift, int scale, bool planes) {
    if (planes)
      klaunch(dit_norm_planes_kernel, gn, dim3(32 * DIT_LN_WARPS), (size_t)0, a, lda, fl, y, ada, k.ald, gate * H, shift * H, scale * H, 1e-5f,
              k.Hb, k.N, pl.N.hi, pl.N.lo, r.lens, r.offs, H);
    else
      klaunch(dit_norm_kernel, gn, dim3(32 * DIT_LN_WARPS), (size_t)0, a, lda, fl, y, ada, k.ald, gate * H, shift * H, scale * H, 1e-5f, k.Hb, k.N,
              r.lens, r.offs, H);
    CK(cudaGetLastError());
    ++launches;
  };
  // one conv of the block: on the tensor cores from the planes `in` when `tc`, else on the FFMA pipe from the fp32 rows x;
  // `out`: the planes of y its consumer reads (or null)
  auto cv = [&](bool tc, const ConvW& W, const TcW& tw, const Planes& in, const float* x, float* y, const Planes* out) {
    if (tc) {
      TcSpec q;
      q.in = in; q.w = tw; q.bias = W.b; q.Cin = W.Cin; q.Cout = W.Cout; q.k = W.k; q.pad = (W.k - 1) / 2;
      q.y = y; q.ldy = W.Cout;
      if (out) q.out = *out;
      launch_tc({q}, 1, r);
    } else {
      ConvP c = mk(W, x, W.Cin, 0, y, W.Cout, 0, 1, (W.k - 1) / 2);
      if (out) { c.p_hi = out->hi; c.p_lo = out->lo; c.ldp = out->C; c.pl_slope = 1.f; }
      launch_conv({c}, 1, r);
    }
  };
  if (tap) st_tap("tc_norm_in", xin, (size_t)H * 4, (size_t)ldi * 4);
  norm(xin, ldi, film, nullptr, 2, 0, 1, p.qkv || p.ffn1);
  if (tap) CK(cudaMemcpyAsync(ensure(d_stdbg_n, T * H), k.N, T * H * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  if (tap && (p.qkv || p.ffn1)) st_tap_planes("tc_norm_hi", "tc_norm_lo", pl.N, H, H);
  cv(p.qkv, L.qkv, L.t_qkv, pl.N, k.N, k.QKV, attn_tc ? &pl.QKV : nullptr);
  if (tap) st_tap("tc_qkv_in", k.QKV, (size_t)3 * H * 4, (size_t)3 * H * 4);
  if (attn_tc)
    klaunch(dit_rope_planes_kernel, gs, dim3(128), (size_t)0, k.QKV, k.rope, k.heads, dk, k.rd, pl.QKV.hi, pl.QKV.lo, r.lens, r.offs);
  else
    klaunch(dit_rope_kernel, gs, dim3(128), (size_t)0, k.QKV, k.rope, k.heads, dk, k.rd, r.lens, r.offs);
  CK(cudaGetLastError());
  ++launches;
  if (tap) CK(cudaMemcpyAsync(ensure(d_stdbg_qkv, T * 3 * H), k.QKV, T * 3 * H * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  if (tap && attn_tc) st_tap_planes("tc_qkv_hi", "tc_qkv_lo", pl.QKV, 3 * H, 3 * H);
  Planes* pao = p.o ? const_cast<Planes*>(&pl.AO) : nullptr;
  if (attn_tc) launch_attn_tc(pl.QKV, k.AO, pao, L, H, r);
  else launch_attn(k.QKV, k.AO, L, H, pao, r);
  cv(p.o, L.o, L.t_o, pl.AO, k.AO, k.Y, nullptr);
  norm(k.Hb, H, nullptr, k.Y, 2, 3, 4, p.ffn1);
  cv(p.ffn1, L.ffn1, L.t_ffn1, pl.N, k.N, k.FF, nullptr);
  if (tap) st_tap("tc_silu_in", k.FF, (size_t)F * 4, (size_t)F * 4);
  if (p.ffn2)
    klaunch(dit_silu_planes_kernel, gs, dim3(256), (size_t)0, k.FF, F, pl.FF.hi, pl.FF.lo, r.lens, r.offs);
  else
    klaunch(dit_silu_kernel, gs, dim3(256), (size_t)0, k.FF, F, r.lens, r.offs);
  CK(cudaGetLastError());
  ++launches;
  if (tap) st_tap("tc_silu", k.FF, (size_t)F * 4, (size_t)F * 4);
  if (tap && p.ffn2) st_tap_planes("tc_silu_hi", "tc_silu_lo", pl.FF, F, F);
  cv(p.ffn2, L.ffn2, L.t_ffn2, pl.FF, k.FF, k.Y, nullptr);
  if (tap) { st_tap("tc_gate_x", k.Hb, (size_t)H * 4, (size_t)H * 4); st_tap("tc_gate_y", k.Y, (size_t)H * 4, (size_t)H * 4); }
  if (xout_pl)
    klaunch(dit_gate_planes_kernel, gs, dim3(128), (size_t)0, (const float*)k.Hb, (const float*)k.Y, ada, k.ald, 5 * H, xout, ldo, xout_pl->hi,
            xout_pl->lo, r.lens, r.offs, H);
  else
    klaunch(dit_gate_kernel, gs, dim3(128), (size_t)0, (const float*)k.Hb, (const float*)k.Y, ada, k.ald, 5 * H, xout, ldo, r.lens, r.offs, H);
  CK(cudaGetLastError());
  ++launches;
  if (tap) st_tap("tc_gate", xout, (size_t)H * 4, (size_t)ldo * 4);
  if (tap && xout_pl) st_tap_planes("tc_gate_hi", "tc_gate_lo", *xout_pl, H, ldo);
}

// The whole call: uploads, the hoisted conditioning (FiLM rows of every step, adaLN rows of every sequence, cond_proj of both
// branches, the rotary table), then n Euler steps of the estimator over the ragged batch of both branches.  The step loop is
// unrolled into the enqueue (and so into the call's graph): step k's FiLM rows and dt are addresses, not values.
//
// Every sequence has a length and an extent >= it (rows are packed by extent).  The reference's synthesise pads the frame axis
// to a multiple of 4 and masks only what the blocks write, so the noise, cond_proj and in_proj live on the extent and reach
// the last valid frames through the convs' taps; everything else lives on the length.  vtts_cfm_decode passes extent == length.
void vtts_engine::st_enqueue() {
  const vtts_config& c = cfg;
  const int NC = c.st_noise, MC = c.st_cond, H = c.st_hidden, F = c.st_filter, NL = c.st_layers, G = c.st_spk_dim;
  const int NS = stp.NS, Bu = B, XW = NC + H, dk = H / c.st_heads, rd = dk / 2, nlsc = NL / 2;
  const size_t T = (size_t)stp.Ttot;
  int* di = ensure(d_sti, 4 * NS);
  float* df = ensure(d_stf, ST_PRM + (size_t)Bu * G);
  float* mu = ensure(d_stmu, T * MC);
  float* noise = stp.noise ? ensure(d_stnoise, (size_t)Tfrm * NC) : nullptr;
  stg[STG_ST_MEL].upload();
  const int *lens = di, *offs = di + NS, *sid = di + 2 * NS, *exts = di + 3 * NS;
  const float *prm = df, *ts = df + 16, *dts = df + 16 + VTTS_CFM_MAX_STEPS;
  // The NS sequences in one fixed launch shape for every conv and one attention kernel (Tuning::fixed_ffma, fixed_attention):
  // every row is summed in the same order whatever the batch, so an utterance's mel does not depend on what it is batched with.
  // The heuristics see every sequence at the bucket, the profiler the unconditional branches at their conditional twins' lengths.
  // In precision mode 2 the tensor-core convs run without split-K and the attention on attn_tc_kernel (Tuning::fixed_tc), which
  // keeps that property: each output is summed by one CTA in one k order whatever the launch shape.
  const StPipe& pp_tc = stp_tc;
  Rows rl{lens, offs, NS, maxFrm, std::vector<int>(NS, maxFrm), std::vector<int>(h_frm_len.begin(), h_frm_len.begin() + Bu),
          pp_tc.on ? tune.fixed_ffma().fixed_attention().fixed_tc() : tune.fixed_ffma().fixed_attention()};
  if (stp.guided) rl.real.insert(rl.real.end(), h_frm_len.begin(), h_frm_len.begin() + Bu);
  Rows re = rl;                                     // the same rows over the extents
  re.lens = exts;
  float* film = ensure(d_stfilm, (size_t)VTTS_CFM_MAX_STEPS * NL * 2 * H);
  float* ada = ensure(d_stada, (size_t)NS * NL * 6 * H);
  float2* rope = reinterpret_cast<float2*>(ensure(d_strope, (size_t)maxFrm * rd));
  float *xc = ensure(d_stxc, T * XW), *p0 = ensure(d_stp0, T * F), *p1 = ensure(d_stp1, T * F);
  float* cat[4];
  for (int j = 0; j < nlsc; ++j) cat[j] = ensure(d_stcat[j], T * 2 * H);
  float *X = ensure(d_stx, T * H), *X2 = ensure(d_stx2, T * H);
  StBlk kb{H, F, c.st_heads, rd, NL * 6 * H, rope, ada,
           ensure(d_sth, T * H), ensure(d_stn, T * H), ensure(d_stqkv, T * 3 * H), ensure(d_stao, T * H), ensure(d_sty, T * H), ensure(d_stff, T * F)};
  float *V = ensure(d_stv, T * NC), *mel = ensure(d_stmel, (size_t)Tfrm * NC * (stp.prior ? 2 : 1));
  const dim3 gs(maxFrm, NS);
  // ---- once per call
  if (stp.text) {     // mu rows, pause flags and the prior from the token rows the text phase left on the device
    const int *tl = d_stti.p, *to = tl + Bu, *dur = d_sttd.p, *first = dur + Ttok;
    klaunch(stt_expand_kernel, dim3(maxTok, Bu), dim3(128), (size_t)0, (const float*)d_sttx.p, MC, (const float*)(d_sttf.p + 16), (const float*)d_stmumel.p, NC,
            dur, first, mu, ensure(d_stpau, (size_t)Tfrm), stp.prior ? mel + (size_t)Tfrm * NC : (float*)nullptr, prm, st_mel_mean, st_mel_std, tl, to, offs);
    CK(cudaGetLastError());
    ++launches;
  }
  klaunch(dit_init_kernel, gs, dim3(128), (size_t)0, (const float*)noise, prm, st_fake_content, xc, XW, NC, mu, MC, cat[nlsc - 1], H, lens, exts, offs, Bu);
  klaunch(dit_time_kernel, dim3(stp.steps), dim3(256), (size_t)0, ts, st_tw1, st_tb1, st_tw2, st_tb2, st_fw, st_fb, H, F, NL, film);
  klaunch(dit_ada_kernel, dim3(NL, NS), dim3(256), (size_t)0, st_emb, st_fake_spk, stp.rows ? (const float*)(df + ST_PRM) : (const float*)nullptr,
          sid, st_aw1, st_ab1, st_aw2, st_ab2, G, H, NL, c.st_n_spks, ada);
  klaunch(dit_rope_table_kernel, dim3((maxFrm * (rd / 2) + 127) / 128), dim3(128), (size_t)0, rope, maxFrm, rd);
  CK(cudaGetLastError());
  launches += 4;
  auto silu = [&](float* y, int width) {
    klaunch(dit_silu_kernel, gs, dim3(256), (size_t)0, y, width, exts, offs);
    CK(cudaGetLastError());
    ++launches;
  };
  auto cv = [&](const ConvW& W, const float* x, int ldx, float* y, int ldy, int yoff, const Rows& r) {
    launch_conv({mk(W, x, ldx, 0, y, ldy, yoff, 1, (W.k - 1) / 2)}, 1, r);
  };
  // precision mode 2: the planes of every tensor-core operand (stpl), whose rows behind each sequence's length one
  // zero_tails launch over the NS sequences clears (producers over the extent then write their rows up to it), and a conv
  // on the tensor cores where stp_tc puts it
  const StPipe& pt = pp_tc;
  stpl = StPl{};
  if (pt.on) {
    begin_planes();
    const long R = (long)T;
    int slot = 40;    // plane slots 40.. (the flow's in a VITS2 engine; the vocoder uses 0.., BERT 51..)
    if (pt.cp[0]) stpl.mu = planes(slot++, R, 1, MC);
    if (pt.cp[1]) stpl.p0 = planes(slot++, R, 1, F);
    if (pt.cp[2]) stpl.p1 = planes(slot++, R, 1, F);
    if (pt.qkv || pt.ffn1) stpl.N = planes(slot++, R, 1, H);
    if (pt.attn) stpl.QKV = planes(slot++, R, 1, 3 * H);
    if (pt.o) stpl.AO = planes(slot++, R, 1, H);
    if (pt.ffn2) stpl.FF = planes(slot++, R, 1, F);
    for (int j = 0; j < nlsc && pt.lsc; ++j) stpl.cat[j] = planes(slot++, R, 1, 2 * H);
    collecting = false;
    if (tail.n) {
      klaunch(zero_tails_kernel, dim3(tail.n, NS), dim3(128), (size_t)0, tail, lens, offs, NS);
      CK(cudaGetLastError());
      ++launches;
    }
  }
  auto cvt = [&](bool tc, const ConvW& W, const TcW& tw, const Planes& in, const float* x, int ldx, float* y, int ldy, int yoff, const Planes* out,
                 int poff, const Rows& r) {
    if (!tc) {
      ConvP p = mk(W, x, ldx, 0, y, ldy, yoff, 1, (W.k - 1) / 2);
      if (out) { p.p_hi = out->hi + poff; p.p_lo = out->lo + poff; p.ldp = out->C; p.pl_slope = 1.f; }
      launch_conv({p}, 1, r);
      return;
    }
    TcSpec q;
    q.in = in; q.w = tw; q.bias = W.b; q.Cin = W.Cin; q.Cout = W.Cout; q.k = W.k; q.pad = (W.k - 1) / 2;
    q.y = y; q.ldy = ldy; q.yoff = yoff;
    if (out) { q.out = *out; q.poff = poff; }
    launch_tc({q}, 1, r);
  };
  auto silu_pl = [&](float* y, int width, const Planes& pl) {
    klaunch(dit_silu_planes_kernel, gs, dim3(256), (size_t)0, y, width, pl.hi, pl.lo, exts, offs);
    CK(cudaGetLastError());
    ++launches;
  };
  // cond_proj (decoder.py:121; not masked: zero padded at the ends of each sequence's extent) into the cond columns of the
  // in_proj operand
  if (!pt.on) {
    cv(st_cp[0], mu, MC, p0, F, 0, re);
    silu(p0, F);
    cv(st_cp[1], p0, F, p1, F, 0, re);
    silu(p1, F);
    cv(st_cp[2], p1, F, xc, XW, NC, re);
  } else {
    if (pt.cp[0]) {     // mu's planes over the extents (dit_init_kernel wrote the padding rows)
      klaunch(split_planes_kernel, dim3((maxFrm + EW_ROWS - 1) / EW_ROWS, NS), dim3(EW_THREADS), (size_t)0, (const float*)mu, MC, stpl.mu.hi,
              stpl.mu.lo, MC, MC, 1.f, 0, 1, exts, offs);
      CK(cudaGetLastError());
      ++launches;
    }
    cvt(pt.cp[0], st_cp[0], st_tcp[0], stpl.mu, mu, MC, p0, F, 0, nullptr, 0, re);
    if (pt.cp[1]) silu_pl(p0, F, stpl.p0);
    else silu(p0, F);
    cvt(pt.cp[1], st_cp[1], st_tcp[1], stpl.p0, p0, F, p1, F, 0, nullptr, 0, re);
    if (pt.cp[2]) silu_pl(p1, F, stpl.p1);
    else silu(p1, F);
    cvt(pt.cp[2], st_cp[2], st_tcp[2], stpl.p1, p1, F, xc, XW, NC, nullptr, 0, re);
  }
  // DitWrapper (decoder.py:15-18) of block l at step s; pl: the planes of xout's column block (mode 2), or null
  auto block = [&](int l, int s, const float* xin, int ldi, float* xout, int ldo, const Planes* pl) {
    const bool tap = (debug_flags & 1) && l == 0 && s == 0;
    if (pt.on) st_block_tc(kb, st_blk[l], l, film + ((size_t)s * NL + l) * 2 * H, xin, ldi, xout, ldo, pl, tap, rl);
    else st_block(kb, st_blk[l], l, film + ((size_t)s * NL + l) * 2 * H, xin, ldi, xout, ldo, tap, rl);
  };
  // the planes of column block `half` (0: x, 1: skip) of long-skip operand j, or null on the FFMA pipe
  Planes half_pl[4][2];
  for (int j = 0; j < nlsc && pt.lsc; ++j)
    for (int h = 0; h < 2; ++h) {
      half_pl[j][h] = stpl.cat[j];
      half_pl[j][h].hi += h * H; half_pl[j][h].lo += h * H;
    }
  auto cat_pl = [&](int j, int h) { return pt.lsc ? &half_pl[j][h] : (const Planes*)nullptr; };
  for (int s = 0; s < stp.steps; ++s) {
    // in_proj over (x | cond) (decoder.py:123-124; not masked: over the extent) -> the skip half of the last long-skip operand
    if (pt.lsc) cvt(false, st_in, TcW{}, Planes{}, xc, XW, cat[nlsc - 1], 2 * H, H, &stpl.cat[nlsc - 1], H, re);
    else cv(st_in, xc, XW, cat[nlsc - 1], 2 * H, H, re);
    // blocks 0 .. NL/2-1 leave their input as a skip (decoder.py:130-131): block i reads the skip half of cat[nlsc-1-i] and
    // writes the skip half of the next one; the last of them writes the x half of cat[0]
    for (int i = 0; i < nlsc; ++i)
      block(i, s, cat[nlsc - 1 - i] + H, 2 * H, i + 1 < nlsc ? cat[nlsc - 2 - i] + H : cat[0], 2 * H,
            i + 1 < nlsc ? cat_pl(nlsc - 2 - i, 1) : cat_pl(0, 0));
    // blocks NL/2 ..: the long-skip conv over (x | skip) (decoder.py:133-134), then the block.  The last one's skip is
    // in_proj's output, whose rows past the length its taps read: its input rows are the extent's (the x half is zero there)
    for (int j = 0; j < nlsc; ++j) {
      const bool last = j + 1 == nlsc;
      if (pt.on) cvt(pt.lsc, st_lsc[j], pt.lsc ? st_tlsc[j] : TcW{}, stpl.cat[j], cat[j], 2 * H, X, H, 0, nullptr, 0, last ? re : rl);
      else cv(st_lsc[j], cat[j], 2 * H, X, H, 0, last ? re : rl);
      block(nlsc + j, s, X, H, last ? X2 : cat[j + 1], last ? H : 2 * H, last ? nullptr : cat_pl(j + 1, 0));
    }
    cv(st_final, X2, H, V, NC, 0, rl);
    const bool end = s + 1 == stp.steps;
    klaunch(dit_euler_kernel, dim3(maxFrm, Bu), dim3(128), (size_t)0, (const float*)V, xc, XW, NC, dts + s, prm, stp.guided ? 1 : 0,
            end ? mel : (float*)nullptr, st_mel_mean, st_mel_std, lens, offs, Bu);
    CK(cudaGetLastError());
    ++launches;
  }
  if (stp.text) {
    klaunch(stt_pause_fill_kernel, dim3(maxFrm, Bu), dim3(128), (size_t)0, mel, NC, (const float*)d_stpau.p, lens, offs);
    CK(cudaGetLastError());
    ++launches;
  }
}

// Text phase of vtts_stabletts_synthesise: uploads, the token rows x, dp_encoder and its proj, the durations and their scan;
// with `prior` the mel encoder and its proj as well.  Leaves x, the durations, each token's first frame, the pauses and
// mu_mel on the device for the mel phase, and downloads d_sttd, [dur][first][frames of every utterance] (STG_ST_DURATIONS).  The BERT rows
// are in d_stbert: uploaded with the staged inputs, or gathered there by stt_bert_enqueue.
void vtts_engine::stt_enqueue(bool prior) {
  const vtts_config& c = cfg;
  const int MC = c.st_cond, H = c.st_enc_hidden, F = c.st_enc_filter, NE = c.st_enc_layers, G = c.st_spk_dim, S = c.st_streams;
  const int dk = H / c.st_enc_heads, rd = dk / 2, DC = c.st_dur_channels, NC = c.st_noise;
  const size_t T = (size_t)Ttok, ni = (size_t)3 * B + (size_t)S * T;
  int* di = ensure(d_stti, ni);
  float* df = ensure(d_sttf, 16 + T);
  float* bert = ensure(d_stbert, T * c.st_bert_dim);
  stg[STG_ST_TEXT].upload();
  const int *lens = di, *offs = di + B, *sid = di + 2 * B, *ids = di + 3 * B;
  // the decoder's fixed launch shape, every token row sized at the bucket: durations do not depend on the batch
  const Rows r{lens, offs, B, maxTok, std::vector<int>(B, maxTok), h_tok_len, tune.fixed_ffma().fixed_attention()};
  float* x = ensure(d_sttx, T * MC);
  float2* rope = reinterpret_cast<float2*>(ensure(d_sttrope, (size_t)maxTok * rd));
  float* ada = ensure(d_sttada, (size_t)B * NE * 6 * H);
  float *e0 = ensure(d_stte[0], T * H), *e1 = ensure(d_stte[1], T * H);
  float *mu_mel = ensure(d_stmumel, T * NC), *mu_dp = ensure(d_stmudp, T * DC), *logw = ensure(d_stlogw, T);
  int* dd = ensure(d_sttd, 2 * T + B);
  StBlk kb{H, F, c.st_enc_heads, rd, NE * 6 * H, rope, ada,
           ensure(d_sth, T * H), ensure(d_stn, T * H), ensure(d_stqkv, T * 3 * H), ensure(d_stao, T * H), ensure(d_sty, T * H), ensure(d_stff, T * F)};
  klaunch(stt_front_kernel, dim3(maxTok, B), dim3(256), (size_t)0, ids, Ttok, (const float*)bert, st_tok_emb, (float)std::sqrt((double)c.st_emb_dim),
          st_punc_emb, (float)std::sqrt((double)c.st_punc_dim), st_bert_w, st_bert_b, S, c.st_emb_dim, c.st_punc_dim, c.st_bert_dim, c.st_bert_proj,
          x, lens, offs);
  klaunch(dit_rope_table_kernel, dim3((maxTok * (rd / 2) + 127) / 128), dim3(128), (size_t)0, rope, maxTok, rd);
  CK(cudaGetLastError());
  launches += 2;
  for (int e = prior ? 0 : 1; e < 2; ++e) {
    const StEncW& W = st_enc[e];
    klaunch(dit_ada_kernel, dim3(NE, B), dim3(256), (size_t)0, W.spk, (const float*)nullptr, (const float*)nullptr, sid, W.aw1, W.ab1, W.aw2, W.ab2, G, H,
            NE, c.st_n_spks, ada);
    CK(cudaGetLastError());
    ++launches;
    const float* in = x;
    for (int l = 0; l < NE; ++l) {
      float* out = l % 2 ? e1 : e0;
      st_block(kb, W.blk[l], l, nullptr, in, H, out, H, false, r);
      in = out;
    }
    launch_conv({mk(W.proj, in, H, 0, e == 0 ? mu_mel : mu_dp, e == 0 ? NC : DC, 0, 1, 0)}, 1, r);
  }
  klaunch(stt_dur_kernel, dim3(B), dim3(STT_SCAN), (size_t)0, (const float*)mu_dp, DC, DC, (const float*)(df + 16), (const float*)df,
          (float)VTTS_ST_MAX_TOKEN_FRAMES, dd, dd + Ttok, dd + 2 * Ttok, logw, lens, offs);
  CK(cudaGetLastError());
  ++launches;
  stg[STG_ST_DURATIONS].download();
}

// BERT rows of the text phase from word pieces: BERT of the sentences bt_stage staged, into its packed rows d_btout, then
// st_bert_gather_kernel copies each token's row into d_stbert, where stt_enqueue reads it.  d_stg holds [tok len B][tok off B]
// [source row of every token row Ttok].
void vtts_engine::stt_bert_enqueue() {
  const vtts_config& c = cfg;
  const size_t T = (size_t)Ttok, ni = 2 * (size_t)B + T;
  float* feat = ensure(d_btout, (size_t)btp.tot * c.cv_hidden);
  bt_enqueue(feat);
  int* di = ensure(d_stg, ni);
  float* bert = ensure(d_stbert, T * c.st_bert_dim);
  stg[STG_ST_PIECES].upload();
  klaunch(st_bert_gather_kernel, dim3(maxTok, B), dim3(128), (size_t)0, (const float*)feat, (const int*)(di + 2 * B), c.st_bert_dim, bert,
          (const int*)di, (const int*)(di + B));
  CK(cudaGetLastError());
  ++launches;
}

// Front end (or the caller's log-mel), the three LSTM layers over every slice, and the embedding.  seq: the slice table of
// d_sseq (host copy); max_len: the longest slice.  Not graphed: the slice table is staged here.
void vtts_engine::spk_enqueue(bool from_mel, const std::vector<int>& seq, int max_len) {
  const int ns = spk_nseq;
  Staging& s = stg[STG_SPK_SLICES];
  s.begin();
  s.add(d_sseq, seq.size());
  s.commit();
  std::copy(seq.begin(), seq.end(), s.host(d_sseq));
  s.upload();
  const int* ds = d_sseq.p;
  const int *xrow = ds, *slen = ds + ns, *soff = ds + 2 * ns, *last = ds + 3 * ns + 1, *of_clip = ds + 4 * ns + 1;
  vc_upload(false);
  const float* feat = front_end(from_mel);
  // Sequences per cluster: the fewest that keep every cluster co-resident; more sequences per cluster lengthen each step,
  // more clusters than fit run in waves.
  int NS = 1, li = 0;
  while (NS < 8 && (ns + NS - 1) / NS > spk_clusters[li]) { NS *= 2; ++li; }
  const int groups = (ns + NS - 1) / NS;
  // The projections run with one fixed launch shape (Tuning::fixed_ffma), so every row is summed in the same order whatever
  // the batch: a clip's g does not depend on the clips it is batched with.  Layer 0 runs over the frames, layers 1 and 2 over
  // the slices.
  Rows rf = frm_rows();
  rf.tune = tune.fixed_ffma();
  const std::vector<int> slen_h(seq.begin() + ns, seq.begin() + 2 * ns);
  const Rows rs{slen, soff, ns, max_len, slen_h, slen_h, rf.tune};
  const float* x = feat;
  for (int l = 0; l < 3; ++l) {
    float* xp = ensure(d_sx[l], (size_t)(l == 0 ? Tfrm : spk_rows) * SPK_GATES);
    float* hs = ensure(d_sh[l], (size_t)spk_rows * SPK_H);
    if (l == 0) launch_conv({mk(spk_ih[0], x, spec_pad, 0, xp, SPK_GATES, 0, 1, 0)}, 1, rf);
    else launch_conv({mk(spk_ih[l], x, SPK_H, 0, xp, SPK_GATES, 0, 1, 0)}, 1, rs);
    const int* xr = l == 0 ? xrow : soff;
    const dim3 grid(groups * SPK_CTAS), blk(SPK_THREADS);
    switch (NS) {
      case 1: klaunch(lstm_rec_kernel<1>, grid, blk, spk_rec_smem<1>(), (const float*)xp, spk_hh[l], xr, slen, soff, ns, hs); break;
      case 2: klaunch(lstm_rec_kernel<2>, grid, blk, spk_rec_smem<2>(), (const float*)xp, spk_hh[l], xr, slen, soff, ns, hs); break;
      case 4: klaunch(lstm_rec_kernel<4>, grid, blk, spk_rec_smem<4>(), (const float*)xp, spk_hh[l], xr, slen, soff, ns, hs); break;
      default: klaunch(lstm_rec_kernel<8>, grid, blk, spk_rec_smem<8>(), (const float*)xp, spk_hh[l], xr, slen, soff, ns, hs); break;
    }
    CK(cudaGetLastError());
    ++launches;
    x = hs;
  }
  klaunch(spk_embed_kernel, dim3(B), dim3(SPK_H), (size_t)0, x, last, of_clip, spk_lin_w, spk_lin_b, ensure(d_sg, (size_t)B * SPK_H));
  CK(cudaGetLastError());
  ++launches;
}

// ---------------------------------------------------------------------------------------------------
// QuickVC conversion (SynthesizerTrn.infer, vc/models.py:862-872) from content units and g: cond rows of g, enc_p, the
// reverse flow with g, the decoder with cond(g) and the torch.istft tail.  The frame counts are the unit counts, so the whole
// call is ONE graphed phase.
// ---------------------------------------------------------------------------------------------------
void vtts_engine::quickvc_enqueue(bool eps, bool from_wav) {
  const int G = cfg.gin_channels;
  if (!capturing) CK(cudaEventRecord(ev[4], stream));
  const float* noise = vc_upload(eps);
  const int* fo = d_frm_off.p;
  const Rows r = frm_rows();
  float* units = ensure(d_vin, (size_t)Tfrm * QV_UNITS);       // unit rows, packed as the engine's rows
  if (from_wav) {      // ContentVec writes the unit rows; the gaps between clips and the bucket's tail stay zero
    CK(cudaMemsetAsync(units, 0, (size_t)Tfrm * QV_UNITS * sizeof(float), stream));
    cv_enqueue(units, fo);
  }
  // ---- g's cond rows [B][condR] (the flow's WN cond layers, then dec.cond) in d_condv: the uploaded g rows are the table
  //      cond_vc_kernel reads, through sid_src = b
  float* cond = ensure(d_condv, (size_t)B * condR);
  klaunch(cond_vc_kernel, dim3((condR + 7) / 8, B), dim3(256), (size_t)(G * sizeof(float)), (const float*)d_qg.p,
          (const int*)(d_vint.p + B), cond_w, cond_b, condR, (const float*)nullptr, (const float*)nullptr, 0, cond, (float*)nullptr, G, B, B);
  CK(cudaGetLastError());
  ++launches;
  // ---- z_p, m_p, logs_p = enc_p(c)   (models.py:868)
  posterior_encode(units, QV_UNITS, noise, nullptr, 0, r);
  // ---- z = flow(z_p, g, reverse=True)   (models.py:869)
  float* z = d_z.p;
  const bool flow_on_tc = tc && !flow.empty() && !flow[0].t_in.empty();
  if (flow_on_tc) flow_tc(z, false, cond, condR, /*forward=*/false, r);
  else flow_ffma(z, cond, condR, /*forward=*/false, r);
  if (!capturing) CK(cudaEventRecord(ev[5], stream));
  // ---- o = dec(z * c_mask, g)   (models.py:870)
  decode(z, r);
}

// ===================================================================================================
// C ABI
// ===================================================================================================
namespace {

enum : int { G_ATOMIC = 0, G_BEGIN = 1, G_CONT = 2 };    // one-shot call | opens a two-phase section | continues / closes it

constexpr int ANY_FAMILY = -1;

// family: the model family the entry point serves (VTTS_FAMILY_*), or ANY_FAMILY.
template <typename Fn>
int guarded(vtts_handle h, Fn fn, int mode = G_ATOMIC, int family = VTTS_FAMILY_VITS2) {
  if (!h) return VTTS_ERR_INVALID;
  std::unique_lock<std::mutex> lk(h->mu);
  if (family != ANY_FAMILY && h->cfg.model_family != family) {
    static const char* const names[] = {"VITS2", "QuickVC", "StableTTS", "GPT-SoVITS text-to-semantic", "GPT-SoVITS SoVITS"};
    h->err = std::string("this entry point serves ") + names[family] + " models; the engine holds a " + names[h->cfg.model_family] + " model";
    return VTTS_ERR_INVALID;
  }
  const std::thread::id me = std::this_thread::get_id();
  if (mode == G_CONT) {
    if (!h->two_phase || h->owner != me) {
      h->err = "second phase called without a preceding vtts_durations by the same thread";
      return VTTS_ERR_STATE;
    }
  } else if (h->two_phase && h->owner != me) {
    if (!h->cv.wait_for(lk, std::chrono::seconds(60), [&] { return !h->two_phase; })) {
      h->err = "another thread has held this handle between vtts_durations and vtts_synthesize for 60 s";
      return VTTS_ERR_STATE;
    }
  }
  auto close = [&] { if (h->two_phase) { h->two_phase = false; h->cv.notify_all(); } };
  if (mode != G_CONT) close();          // (the owner itself starting over)
  try {
    cudaError_t e = cudaSetDevice(h->device);
    if (e != cudaSuccess) throw Err{VTTS_ERR_CUDA, std::string("cudaSetDevice: ") + cudaGetErrorString(e)};
    fn();
    if (mode == G_BEGIN) { h->two_phase = true; h->owner = me; }
    if (mode == G_CONT) close();
    return VTTS_OK;
  } catch (const Err& e) {
    h->err = e.msg;
    cudaGetLastError();
    if (mode == G_CONT && e.code != VTTS_ERR_CAPACITY) close();     // a capacity error keeps the durations for a retry
    return e.code;
  } catch (const std::exception& e) {
    h->err = e.what();
    if (mode == G_CONT) close();
    return VTTS_ERR_INVALID;
  }
}

void collect_timings(vtts_handle h) {
  // ev: 0 start, 1 after H2D, 2 after encoder, 3 after dp, 4 phase2 start, 5 after flow, 6 after decoder, 7 after D2H
  float t;
  if (h->last_graphed) {      // stage events are not recorded inside captured graphs
    for (float& v : h->stage_ms) v = 0.f;
    cudaGetLastError();
    return;
  }
  cudaEventElapsedTime(&t, h->ev[1], h->ev[2]); h->stage_ms[0] = t;
  cudaEventElapsedTime(&t, h->ev[2], h->ev[3]); h->stage_ms[1] = t;
  cudaEventElapsedTime(&t, h->ev[4], h->ev[5]); h->stage_ms[2] = t;
  cudaEventElapsedTime(&t, h->ev[5], h->ev[6]); h->stage_ms[3] = t;
  cudaEventElapsedTime(&t, h->ev[0], h->ev[1]); h->stage_ms[4] = t;
  cudaEventElapsedTime(&t, h->ev[6], h->ev[7]); h->stage_ms[5] = t;
}

// Readback of one output field of a call (STG_OUT): the n values of src from element `at`, in a field with room for `room`
// values (a bucket's, so that the block does not grow with every new length).  Returns the values.
template <typename T>
const T* read_back(vtts_handle h, Buf<T>& src, size_t n, size_t room = 0, size_t at = 0) {
  vtts_engine::Staging& s = h->stg[vtts_engine::STG_OUT];
  s.begin();
  s.add(src, n, at, room);
  s.commit();
  s.download_and_wait();
  return s.host(src);
}

// Clip b's lens[b] rows of `width` values from packed row offs[b] of a call's read-back rows to out + b * out_ld.  The rest
// of each output row is left as it is.
template <typename T>
void read_clips(const T* rows, const int* offs, const std::vector<int>& lens, int width, T* out, int64_t out_ld) {
  for (size_t b = 0; b < lens.size(); ++b)
    memcpy(out + b * out_ld, rows + (size_t)offs[b] * width, (size_t)lens[b] * width * sizeof(T));
}

void setup_lengths(vtts_handle h, const int64_t* lengths, int B, int t_max) {
  REQUIRE(B >= 1 && B <= 16384 && t_max >= 1, VTTS_ERR_INVALID, "bad batch size / t_max");
  h->B = B;
  h->h_tok_len.resize(B);
  for (int b = 0; b < B; ++b) {
    REQUIRE(lengths[b] >= 1 && lengths[b] <= t_max, VTTS_ERR_INVALID, "input_lengths must be in [1, t_max]");
    h->h_tok_len[b] = (int)lengths[b];
  }
  vtts_engine::pack_rows(h->h_tok_len, h->h_tok_off);
  h->set_token_shape();
  h->have_durations = false;
  h->have_latent = false;
}

}  // namespace

namespace {

static bool spec_ok(vtts_handle h, int B);
static void enqueue_phase1_host(vtts_handle h, const int64_t* ids, const int64_t* lengths, const int64_t* sid, int B, int t_max,
                               const float* scales, const float* noise_dp, uint64_t seed, bool may_speculate) {
  setup_lengths(h, lengths, B, t_max);
  memcpy(h->scales, scales, 3 * sizeof(float));
  h->seed = seed;
  h->spec_cap = (may_speculate && spec_ok(h, B)) ? vtts_engine::bucket_frm(h->spec_predict()) : 0;
  h->stage_tokens(ids, t_max, true, noise_dp != nullptr);
  int* ps = h->stg[vtts_engine::STG_TOKENS].host(h->d_sid);
  for (int b = 0; b < B; ++b) {
    REQUIRE(!h->has_g || (sid[b] >= 0 && sid[b] < h->cfg.n_speakers), VTTS_ERR_INVALID, "speaker id out of range [0, n_speakers)");
    ps[b] = (int)sid[b];
  }
  h->stage1(t_max, noise_dp);
  h->run_graphed({vtts_engine::TAG_PHASE1, B, h->maxTok, h->Ttok, noise_dp ? 1 : 0},
                 [&] { h->phase1(nullptr, t_max, nullptr, noise_dp, false); });
}

static void impl_durations(vtts_handle h, const int64_t* ids, const int64_t* lengths, const int64_t* sid, int B, int t_max,
                   const float* scales, const float* noise_dp, uint64_t seed, int64_t* y_lengths, int32_t* durations) {
  enqueue_phase1_host(h, ids, lengths, sid, B, t_max, scales, noise_dp, seed, false);
  h->finish1();
  if (B == 1) h->spec_learn();
  for (int b = 0; b < B; ++b) y_lengths[b] = h->h_frm_len[b];
  if (durations) {
    const int* wc = read_back(h, h->d_wceil, h->Ttok);
    for (int b = 0; b < B; ++b) {
      for (int t = 0; t < t_max; ++t)
        durations[(size_t)b * t_max + t] = t < h->h_tok_len[b] ? wc[h->h_tok_off[b] + t] : 0;
    }
  }
}

static void impl_synthesize(vtts_handle h, const float* noise_z, int z_ld, float* wav, int64_t wav_ld, int32_t* frame_token, int idx_ld) {
  REQUIRE(h->have_durations, VTTS_ERR_STATE, "vtts_synthesize called without vtts_durations");
  REQUIRE((int64_t)h->real_maxFrm * h->hop <= wav_ld, VTTS_ERR_CAPACITY, "wav_ld is smaller than hop * max(y_lengths)");
  REQUIRE(!noise_z || z_ld >= h->real_maxFrm, VTTS_ERR_CAPACITY, "noise_z has fewer columns than max(y_lengths)");
  REQUIRE(!frame_token || idx_ld >= h->real_maxFrm, VTTS_ERR_CAPACITY, "frame_token has fewer columns than max(y_lengths)");
  if (noise_z) h->stage_noise_z(noise_z, z_ld);
  // graph key = the length BUCKETS (token rows, frame rows), not the lengths: kernels read the true lengths on the device
  h->run_graphed({vtts_engine::TAG_PHASE2, h->B, h->maxFrm, h->Tfrm, noise_z ? 1 : 0}, [&] { h->phase2(noise_z, z_ld, false); });
  vtts_engine::Staging& s = h->stg[vtts_engine::STG_OUT];
  s.begin();
  if (frame_token) s.add(h->d_ftok, h->real_Tfrm, 0, h->Tfrm);
  s.add(h->d_wav, (size_t)h->real_Tfrm * h->hop, 0, (size_t)h->Tfrm * h->hop);
  s.commit();
  s.download_and_wait();
  if (frame_token) read_clips(s.host(h->d_ftok), h->h_frm_off.data(), h->h_frm_len, 1, frame_token, idx_ld);
  read_clips(s.host(h->d_wav), h->h_frm_off.data(), h->h_frm_len, h->hop, wav, wav_ld);
  collect_timings(h);
  h->have_durations = false;
}

static void enqueue_phase1_dev(vtts_handle h, const int64_t* d_ids, const int64_t* lengths_host, const int64_t* d_sid, int B, int t_max,
                              const float* scales, const float* d_noise_dp, uint64_t seed, bool may_speculate) {
  setup_lengths(h, lengths_host, B, t_max);
  memcpy(h->scales, scales, 3 * sizeof(float));
  h->seed = seed;
  h->spec_cap = (may_speculate && spec_ok(h, B)) ? vtts_engine::bucket_frm(h->spec_predict()) : 0;
  h->stage_tokens(nullptr, t_max, true, false);
  h->stage1(t_max, nullptr);
  h->eps_dp_ld = t_max;      // device noise is read in the caller's [B][2][t_max] layout
  h->run_graphed({vtts_engine::TAG_PHASE1_DEV, B, h->maxTok, h->Ttok, t_max, (long long)(uintptr_t)d_ids, (long long)(uintptr_t)d_sid,
                  (long long)(uintptr_t)d_noise_dp},
                 [&] { h->phase1(d_ids, t_max, d_sid, d_noise_dp, true); });
}

static void impl_durations_dev(vtts_handle h, const int64_t* d_ids, const int64_t* lengths_host, const int64_t* d_sid, int B, int t_max,
                       const float* scales, const float* d_noise_dp, uint64_t seed, int64_t* y_lengths_host) {
  enqueue_phase1_dev(h, d_ids, lengths_host, d_sid, B, t_max, scales, d_noise_dp, seed, false);
  h->finish1();
  if (B == 1) h->spec_learn();
  for (int b = 0; b < B; ++b) y_lengths_host[b] = h->h_frm_len[b];
}

static void impl_synthesize_dev(vtts_handle h, const float* d_noise_z, int z_ld, float* d_wav, int64_t wav_ld);

static bool spec_ok(vtts_handle h, int B) {
  return B == 1 && h->use_spec && h->use_poll && h->spec_ratio > 0.f && !h->profiling && !h->debug_flags;
}

// Both phases of one call through host buffers (vtts_infer).
static void impl_infer(vtts_handle h, const int64_t* ids, const int64_t* lengths, const int64_t* sid, int B, int t_max, const float* scales,
                       const float* noise_dp, const float* noise_z, int z_ld, uint64_t seed, int64_t* y_lengths, float* wav, int64_t wav_ld,
                       int32_t* frame_token, int idx_ld, int* phase) {
  auto now_us = [] { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  const double t_0 = now_us();
  enqueue_phase1_host(h, ids, lengths, sid, B, t_max, scales, noise_dp, seed, true);
  const double t_1 = now_us();
  for (double& v : h->host_us) v = 0.0;
  h->host_us[0] = t_1 - t_0;
  if (h->spec_cap > 0) {
    h->assume_frames(h->spec_cap);
    const int cap = h->maxFrm;
    if (noise_z) h->stage_noise_z(noise_z, z_ld);
    h->run_graphed({vtts_engine::TAG_PHASE2, h->B, h->maxFrm, h->Tfrm, noise_z ? 1 : 0}, [&] { h->phase2(noise_z, z_ld, false); });
    // the true length is not known on the host yet: the bucket's worth of samples comes back
    vtts_engine::Staging& s = h->stg[vtts_engine::STG_OUT];
    s.begin();
    s.add(h->d_wav, (size_t)cap * h->hop);
    if (frame_token) s.add(h->d_ftok, cap);
    s.commit();
    s.download();
    const double t_2 = now_us();
    CK(cudaStreamSynchronize(h->stream));
    const double t_3 = now_us();
    h->host_us[1] = t_2 - t_1; h->host_us[2] = t_3 - t_2;
    REQUIRE(h->read_published_lengths(), VTTS_ERR_CUDA, "phase 1 finished without publishing the utterance lengths");
    const int real = h->h_frm_len[0];
    h->real_Tfrm = real; h->real_maxFrm = real;
    h->spec_learn();
    y_lengths[0] = real;
    *phase = 1;
    h->host_us[5] = real <= cap ? 1.0 : 2.0;
    if (real <= cap) {
      ++h->spec_hits;
      h->last_graphed = true;
      h->have_durations = true;          // (kept if one of the capacity checks below fails)
      REQUIRE((int64_t)real * h->hop <= wav_ld, VTTS_ERR_CAPACITY, "wav_ld is smaller than hop * max(y_lengths)");
      REQUIRE(!noise_z || z_ld >= real, VTTS_ERR_CAPACITY, "noise_z has fewer columns than max(y_lengths)");
      REQUIRE(!frame_token || idx_ld >= real, VTTS_ERR_CAPACITY, "frame_token has fewer columns than max(y_lengths)");
      memcpy(wav, s.host(h->d_wav), (size_t)real * h->hop * sizeof(float));
      if (frame_token) memcpy(frame_token, s.host(h->d_ftok), (size_t)real * sizeof(int));
      h->have_durations = false;
      h->host_us[3] = now_us() - t_3; h->host_us[4] = now_us() - t_0;
      return;
    }
    ++h->spec_misses;                    // predicted bucket too small (the device-side lengths were clamped to it): true
    h->set_frame_shape();                //   lengths back, second phase again with the real shape
    h->klaunch(restore_lengths_kernel, dim3(1), dim3(32), (size_t)0, (const int*)h->d_frm_len_real.p, h->d_frm_len.p, h->d_frm_off.p, h->B);
    h->have_durations = true;
  } else {
    h->finish1();
    if (B == 1) h->spec_learn();
    for (int b = 0; b < B; ++b) y_lengths[b] = h->h_frm_len[b];
    *phase = 1;
  }
  impl_synthesize(h, noise_z, z_ld, wav, wav_ld, frame_token, idx_ld);
}

// Both phases through device buffers (vtts_infer_dev).
static void impl_infer_dev(vtts_handle h, const int64_t* d_ids, const int64_t* lengths_host, const int64_t* d_sid, int B, int t_max,
                           const float* scales, const float* d_noise_dp, const float* d_noise_z, int z_ld, uint64_t seed,
                           int64_t* y_lengths_host, float* d_wav, int64_t wav_ld, int* phase) {
  enqueue_phase1_dev(h, d_ids, lengths_host, d_sid, B, t_max, scales, d_noise_dp, seed, true);
  if (h->spec_cap > 0) {
    h->assume_frames(h->spec_cap);
    const int cap = h->maxFrm;
    h->run_graphed({vtts_engine::TAG_PHASE2_DEV, h->B, h->maxFrm, h->Tfrm, z_ld, (long long)(uintptr_t)d_noise_z}, [&] { h->phase2(d_noise_z, z_ld, true); });
    const size_t ncopy = (size_t)std::min<int64_t>((int64_t)cap * h->hop, wav_ld);
    CK(cudaMemcpyAsync(d_wav, h->d_wav.p, ncopy * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    REQUIRE(h->read_published_lengths(), VTTS_ERR_CUDA, "phase 1 finished without publishing the utterance lengths");
    const int real = h->h_frm_len[0];
    h->real_Tfrm = real; h->real_maxFrm = real;
    h->spec_learn();
    y_lengths_host[0] = real;
    *phase = 1;
    if (real <= cap) {
      ++h->spec_hits;
      h->last_graphed = true;
      h->have_durations = true;
      REQUIRE((int64_t)real * h->hop <= wav_ld, VTTS_ERR_CAPACITY, "wav_ld is smaller than hop * max(y_lengths)");
      REQUIRE(!d_noise_z || z_ld >= real, VTTS_ERR_CAPACITY, "noise_z has fewer columns than max(y_lengths)");
      h->have_durations = false;
      return;
    }
    ++h->spec_misses;
    h->set_frame_shape();
    h->klaunch(restore_lengths_kernel, dim3(1), dim3(32), (size_t)0, (const int*)h->d_frm_len_real.p, h->d_frm_len.p, h->d_frm_off.p, h->B);
    h->have_durations = true;
  } else {
    h->finish1();
    if (B == 1) h->spec_learn();
    for (int b = 0; b < B; ++b) y_lengths_host[b] = h->h_frm_len[b];
    *phase = 1;
  }
  impl_synthesize_dev(h, d_noise_z, z_ld, d_wav, wav_ld);
}

// Frame shape of a call on recordings (vtts_convert*, vtts_align*): frames per clip from the sample / spectrogram lengths.
static std::vector<int> clip_frames(vtts_handle h, bool from_spec, const int64_t* lengths, int B, int64_t ld) {
  const vtts_config& c = h->cfg;
  REQUIRE(B >= 1 && B <= 16384 && ld >= 1, VTTS_ERR_INVALID, "bad batch size / row pitch");
  std::vector<int> frames(B);
  for (int b = 0; b < B; ++b) {
    const int64_t L = lengths[b];
    if (from_spec) {
      REQUIRE(L >= 1 && L <= ld, VTTS_ERR_INVALID, "spec_lengths must be in [1, spec_ld]");
      frames[b] = (int)L;
    } else {
      REQUIRE(L <= ld, VTTS_ERR_INVALID, "wav_lengths must not exceed wav_ld");
      // the reflect padding needs L > pad, and one frame needs L + 2 * pad >= filter_length, i.e. L >= hop_length
      const int64_t min_len = std::max<int64_t>(h->vc_pad + 1, c.hop_length);
      REQUIRE(L >= min_len, VTTS_ERR_INVALID, "clip too short: the spectrogram needs at least " + std::to_string(min_len) +
              " samples (more than the reflect padding of " + std::to_string(h->vc_pad) + ", and one frame)");
      REQUIRE(L < (1LL << 30), VTTS_ERR_INVALID, "clip too long");
      frames[b] = (int)((L + 2 * h->vc_pad - c.filter_length) / c.hop_length + 1);
    }
  }
  return frames;
}

// Sets the frame shape and stages the recordings, speaker ids (sid_tgt may be null), noise and scalars (stage_clip_fields).
static void stage_clips(vtts_handle h, bool from_spec, const float* in, const int64_t* lengths, int64_t ld, const std::vector<int>& frames,
                        const int64_t* sid_src, const int64_t* sid_tgt, float noise_scale, const float* noise_q, int q_ld, uint64_t seed) {
  const vtts_config& c = h->cfg;
  const int B = h->B;
  h->pack_frames(frames);
  h->vc_wld = (h->maxFrm + 2) * c.hop_length + c.filter_length;
  const int maxF = h->maxFrm, C = c.spec_channels;
  h->stage_clip_fields(from_spec ? vtts_engine::IN_SPEC : vtts_engine::IN_WAV, noise_q != nullptr);
  vtts_engine::Staging& s = h->stg[vtts_engine::STG_CLIPS];
  memcpy(s.host(h->d_frm_len), frames.data(), B * sizeof(int));
  memcpy(s.host(h->d_frm_off), h->h_frm_off.data(), (B + 1) * sizeof(int));
  int* vi = s.host(h->d_vint);
  float* pin = s.host(h->d_vin);
  for (int b = 0; b < B; ++b) {
    vi[b] = (int)lengths[b];
    vi[B + b] = sid_src ? (int)sid_src[b] : 0;
    vi[2 * B + b] = sid_tgt ? (int)sid_tgt[b] : 0;
    if (from_spec) {
      for (int ch = 0; ch < C; ++ch)
        memcpy(pin + ((size_t)b * C + ch) * maxF, in + ((size_t)b * C + ch) * ld, (size_t)frames[b] * sizeof(float));
    } else {
      memcpy(pin + (size_t)b * h->vc_wld, in + (size_t)b * ld, (size_t)lengths[b] * sizeof(float));
    }
  }
  if (noise_q) h->stage_noise(s.host(h->d_vnoise), noise_q, q_ld, frames);
  vtts_engine::put_scalars(s.host(h->d_vprm), 16, &noise_scale, 1, seed);
}

// Voice conversion through host buffers (vtts_convert / vtts_convert_spec).
static void impl_convert(vtts_handle h, bool from_spec, const float* in, const int64_t* lengths, int B, int64_t ld,
                         const int64_t* sid_src, const int64_t* sid_tgt, float noise_scale, const float* noise_q, int q_ld,
                         uint64_t seed, float* out_wav, int64_t out_ld, int64_t* out_frames) {
  const vtts_config& c = h->cfg;
  REQUIRE(c.flow_n_flows % 2 == 0, VTTS_ERR_INVALID, "voice conversion needs an even flow_n_flows (the Flip folding of the packed "
          "flow holds for both directions only then)");
  REQUIRE(h->has_encq, VTTS_ERR_INVALID, "the weight blob has no posterior encoder (enc_q): voice conversion needs a model packed "
          "with posterior=True from a training checkpoint (model.onnx does not contain enc_q)");
  REQUIRE(h->has_g && c.n_speakers > 1, VTTS_ERR_INVALID, "voice conversion needs a multi-speaker model (n_speakers > 1)");
  const std::vector<int> frames = clip_frames(h, from_spec, lengths, B, ld);
  for (int b = 0; b < B; ++b)
    REQUIRE(sid_src[b] >= 0 && sid_src[b] < c.n_speakers && sid_tgt[b] >= 0 && sid_tgt[b] < c.n_speakers, VTTS_ERR_INVALID,
            "speaker id out of range [0, n_speakers)");
  h->B = B;
  h->have_durations = false;
  h->have_latent = false;
  const int real_max = *std::max_element(frames.begin(), frames.end());
  REQUIRE((int64_t)real_max * h->hop <= out_ld, VTTS_ERR_CAPACITY, "out_ld is smaller than hop * max(frames)");
  REQUIRE(!noise_q || q_ld >= real_max, VTTS_ERR_CAPACITY, "noise_q has fewer columns than max(frames)");
  stage_clips(h, from_spec, in, lengths, ld, frames, sid_src, sid_tgt, noise_scale, noise_q, q_ld, seed);
  h->run_graphed({vtts_engine::TAG_CONVERT, B, h->maxFrm, h->Tfrm, from_spec ? 1 : 0, noise_q ? 1 : 0},
                 [&] { h->convert_enqueue(from_spec, noise_q != nullptr); });
  read_clips(read_back(h, h->d_wav, (size_t)h->real_Tfrm * h->hop, (size_t)h->Tfrm * h->hop), h->h_frm_off.data(), frames, h->hop,
             out_wav, out_ld);
  std::copy(frames.begin(), frames.end(), out_frames);
}

// QuickVC speaker embedding through host buffers (vtts_speaker_embedding / _mel).
static void impl_speaker_embedding(vtts_handle h, bool from_mel, const float* in, const int64_t* lengths, int B, int64_t ld, float* g_out) {
  const std::vector<int> frames = clip_frames(h, from_mel, lengths, B, ld);
  h->B = B;
  stage_clips(h, from_mel, in, lengths, ld, frames, nullptr, nullptr, 0.f, nullptr, 0, 0);
  // slices of embed_utterance (vc/models.py:739-760): T <= 128 frames -> the whole clip; else starts 0, 64, ... < T - 128
  // and the last 128 frames.  Slice rows are packed in clip order with SEQ_GAP rows between slices.
  std::vector<int> xrow, slen, soff, last, of_clip(1, 0);
  int off = 0, max_len = 0;
  for (int b = 0; b < B; ++b) {
    const int T = frames[b];
    std::vector<int> starts;
    if (T <= SPK_SLICE) starts.push_back(0);
    else {
      for (int s = 0; s < T - SPK_SLICE; s += SPK_HOP) starts.push_back(s);
      starts.push_back(T - SPK_SLICE);
    }
    for (int s : starts) {
      const int L = std::min(T, SPK_SLICE);
      xrow.push_back(h->h_frm_off[b] + s);
      slen.push_back(L);
      soff.push_back(off);
      last.push_back(off + L - 1);
      off += L + SEQ_GAP;
      max_len = std::max(max_len, L);
    }
    of_clip.push_back((int)xrow.size());
  }
  const int ns = (int)xrow.size();
  h->spk_nseq = ns;
  h->spk_rows = off;
  soff.push_back(off);
  std::vector<int> seq;
  for (auto* v : {&xrow, &slen, &soff, &last, &of_clip}) seq.insert(seq.end(), v->begin(), v->end());
  h->spk_enqueue(from_mel, seq, max_len);
  memcpy(g_out, read_back(h, h->d_sg, (size_t)B * SPK_H), (size_t)B * SPK_H * sizeof(float));
}

// Forced alignment through host buffers (vtts_align / vtts_align_spec).
static void impl_align(vtts_handle h, bool from_spec, const int64_t* ids, const int64_t* id_lengths, int t_max, const int64_t* sid,
                       const float* in, const int64_t* lengths, int B, int64_t ld, float noise_scale, const float* noise_q, int q_ld,
                       uint64_t seed, int32_t* durations, int32_t* token_of_frame, int64_t tof_ld, float* score, int64_t* out_frames) {
  const vtts_config& c = h->cfg;
  REQUIRE(c.flow_n_flows % 2 == 0, VTTS_ERR_INVALID, "alignment needs an even flow_n_flows (the Flip folding of the packed flow holds "
          "for the forward direction only then)");
  REQUIRE(h->has_encq, VTTS_ERR_INVALID, "the weight blob has no posterior encoder (enc_q): alignment needs a model packed with "
          "pack(posterior=True) / Model(voice_conversion=True) from a training checkpoint (model.onnx does not contain enc_q)");
  REQUIRE(t_max >= 1, VTTS_ERR_INVALID, "bad t_max");
  const std::vector<int> frames = clip_frames(h, from_spec, lengths, B, ld);
  constexpr int TX_MAX = MAS_THREADS * MAS_MAXPT;
  for (int b = 0; b < B; ++b) {
    const int64_t tx = id_lengths[b];
    REQUIRE(tx >= 1, VTTS_ERR_INVALID, "id_lengths must be at least 1: an utterance without tokens has no alignment");
    REQUIRE(tx <= t_max, VTTS_ERR_INVALID, "id_lengths must not exceed t_max");
    REQUIRE(tx <= TX_MAX, VTTS_ERR_INVALID, "more than " + std::to_string(TX_MAX) + " tokens in one utterance: above the alignment's limit");
    REQUIRE(tx <= frames[b], VTTS_ERR_INVALID, "more tokens (" + std::to_string(tx) + ") than frames (" + std::to_string(frames[b]) +
            ") in utterance " + std::to_string(b) + ": no monotonic alignment exists");
    REQUIRE(!h->has_g || (sid && sid[b] >= 0 && sid[b] < c.n_speakers), VTTS_ERR_INVALID, "speaker id out of range [0, n_speakers)");
  }
  const int real_max = *std::max_element(frames.begin(), frames.end());
  REQUIRE(!token_of_frame || tof_ld >= real_max, VTTS_ERR_CAPACITY, "tof_ld is smaller than max(frames)");
  REQUIRE(!noise_q || q_ld >= real_max, VTTS_ERR_CAPACITY, "noise_q has fewer columns than max(frames)");
  setup_lengths(h, id_lengths, B, t_max);
  h->stage_tokens(ids, t_max, false, false);        // (the alignment does not advance phase 1's poll sequence)
  stage_clips(h, from_spec, in, lengths, ld, frames, h->has_g ? sid : nullptr, nullptr, noise_scale, noise_q, q_ld, seed);
  h->run_graphed({vtts_engine::TAG_ALIGN, B, h->maxTok, h->Ttok, h->maxFrm, h->Tfrm, from_spec ? 1 : 0, noise_q ? 1 : 0},
                 [&] { h->align_enqueue(from_spec, noise_q != nullptr); });
  vtts_engine::Staging& s = h->stg[vtts_engine::STG_OUT];
  s.begin();
  s.add(h->d_adur, h->real_Ttok);
  s.add(h->d_atof, h->real_Tfrm);
  s.add(h->d_ascore, B);
  s.commit();
  s.download_and_wait();
  for (int b = 0; b < B; ++b) {
    const int tx = h->h_tok_len[b], ty = frames[b];
    int32_t* d = durations + (size_t)b * t_max;
    memcpy(d, s.host(h->d_adur) + h->h_tok_off[b], (size_t)tx * sizeof(int));
    std::fill(d + tx, d + t_max, 0);
    if (token_of_frame) {
      int32_t* f = token_of_frame + (size_t)b * tof_ld;
      memcpy(f, s.host(h->d_atof) + h->h_frm_off[b], (size_t)ty * sizeof(int));
      std::fill(f + ty, f + tof_ld, -1);
    }
    if (score) score[b] = s.host(h->d_ascore)[b];
    out_frames[b] = ty;
  }
}

// QuickVC conversion through host buffers (vtts_quickvc_convert).
static void require_contentvec(vtts_handle h, int B) {
  REQUIRE(h->has_cv, VTTS_ERR_INVALID, "the weight blob has no ContentVec (cv.*): pack it with weights.pack_quickvc(..., contentvec=...)");
  REQUIRE(B >= 1 && B <= 16384, VTTS_ERR_INVALID, "bad batch size");
}

// ContentVec units through host buffers (vtts_content_units).
static void impl_content_units(vtts_handle h, const float* wav, const int64_t* lengths, int B, int64_t wav_ld, float* units,
                               int64_t units_ld, int64_t* out_frames) {
  require_contentvec(h, B);
  REQUIRE(wav_ld >= 1, VTTS_ERR_INVALID, "bad wav_ld");
  h->B = B;
  const std::vector<int> frames = h->cv_stage(wav, lengths, wav_ld);
  for (int b = 0; b < B; ++b) REQUIRE(frames[b] <= units_ld, VTTS_ERR_CAPACITY, "units_ld is smaller than a clip's frame count");
  const int H = h->cfg.cv_hidden, NL = h->cfg.cv_n_conv;
  const size_t Tf = (size_t)h->cvp.tot0 / h->cv_P;
  h->run_graphed({vtts_engine::TAG_CONTENTVEC, B, h->cvp.maxS, h->cvp.tot0}, [&] { h->cv_enqueue(h->ensure(h->d_cvu, Tf * H), nullptr); });
  read_clips(read_back(h, h->d_cvu, Tf * H), h->cvp.h.data() + (NL + NL - 1) * B, frames, H, units, units_ld * H);
  for (int b = 0; b < B; ++b) {
    std::fill(units + ((size_t)b * units_ld + frames[b]) * H, units + (size_t)(b + 1) * units_ld * H, 0.f);
    out_frames[b] = frames[b];
  }
}

// SoVITS semantic codes through host buffers (vtts_sovits_semantic / vtts_sovits_latent): stages the tail, runs it (after
// ContentVec of wav when given) as one graphed phase, and reads each clip's frames / 2 codes back, -1 after them.
static void impl_sovits(vtts_handle h, const float* wav, const float* feats, const int64_t* lengths, int B, int64_t ld,
                        int64_t* codes, int64_t codes_ld, int64_t* out_frames) {
  REQUIRE(B >= 1 && B <= 16384, VTTS_ERR_INVALID, "bad batch size");
  REQUIRE(ld >= 1 && codes_ld >= 0, VTTS_ERR_INVALID, "bad wav_ld / feats_ld / codes_ld");
  h->B = B;
  std::vector<int> frames(B);
  std::vector<long long> key;
  int pairs_cap = 0, maxP = 0;
  if (wav) {
    frames = h->cv_stage(wav, lengths, ld);
    const int NL = h->cfg.cv_n_conv;
    // HuBERT's frame rows of the key's layer-0 rows bound every clip's pair rows (frames + 1 <= its padded rows / cv_P)
    pairs_cap = (h->cvp.tot0 / h->cv_P + 1) / 2;
    maxP = h->cvp.maxL[NL - 1] / 2;
    key = {vtts_engine::TAG_SOVITS, B, h->cvp.maxS, h->cvp.tot0};
  } else {
    for (int b = 0; b < B; ++b) {
      REQUIRE(lengths[b] >= 0 && lengths[b] <= ld, VTTS_ERR_INVALID, "frames must be in [0, feats_ld]");
      frames[b] = (int)lengths[b];
      pairs_cap += (frames[b] + 1) / 2;
      maxP = std::max(maxP, frames[b] / 2);
    }
    pairs_cap = std::max(pairs_cap, 1);
    key = {vtts_engine::TAG_SOVITS_LATENT, B, maxP, pairs_cap};
  }
  for (int b = 0; b < B; ++b) REQUIRE(frames[b] / 2 <= codes_ld, VTTS_ERR_CAPACITY, "codes_ld is smaller than a clip's code count");
  h->sv_stage(frames, pairs_cap, maxP, feats, ld);
  const bool from_wav = wav != nullptr;
  h->run_graphed({key[0], key[1], key[2], key[3]}, [&] { h->sv_enqueue(from_wav); });
  const int* rows = read_back(h, h->d_svcodes, (size_t)pairs_cap);
  for (int b = 0; b < B; ++b) {
    const int n = frames[b] / 2, off = h->svp.h[2 * B + b];
    for (int t = 0; t < n; ++t) codes[(size_t)b * codes_ld + t] = rows[off + t];
    for (int64_t t = n; t < codes_ld; ++t) codes[(size_t)b * codes_ld + t] = -1;
    out_frames[b] = n;
  }
}

// BERT features through host buffers (vtts_bert_features).
static void impl_bert_features(vtts_handle h, const int64_t* ids, const int64_t* lengths, int B, int64_t ids_ld, float* out, int64_t out_ld) {
  REQUIRE(h->has_bert, VTTS_ERR_INVALID, "the weight blob has no BERT (bt.*): build the engine with StableTTS(..., bert=...)");
  REQUIRE(B >= 1 && B <= 16384, VTTS_ERR_INVALID, "bad batch size");
  REQUIRE(ids_ld >= 1, VTTS_ERR_INVALID, "bad ids_ld");
  h->B = B;
  h->bt_stage(ids, lengths, ids_ld);
  for (int b = 0; b < B; ++b) REQUIRE(h->btp.len[b] <= out_ld, VTTS_ERR_CAPACITY, "out_ld is smaller than a sentence's length");
  const int H = h->cfg.cv_hidden;
  const size_t n = (size_t)h->btp.tot * H;
  vtts_engine::Staging& s = h->stg[vtts_engine::STG_OUT];      // listed before the graph captures (growth retires it)
  s.begin();
  s.add(h->d_btout, n);
  s.commit();
  h->run_graphed({vtts_engine::TAG_BERT, B, h->btp.maxL, h->btp.tot}, [&] { h->bt_enqueue(h->ensure(h->d_btout, n)); });
  s.download_and_wait();
  read_clips(s.host(h->d_btout), h->btp.off.data(), h->btp.len, H, out, out_ld * H);
  for (int b = 0; b < B; ++b) std::fill(out + ((size_t)b * out_ld + h->btp.len[b]) * H, out + (size_t)(b + 1) * out_ld * H, 0.f);
}

// Text-to-semantic decoding through host buffers (vtts_t2s_decode).  The text rows run through post_ln_layers once (each
// layer's k, v rows copied into the cache behind its qkv GEMM); then every step runs the layers on one audio token per
// utterance (a prompt token, or the token sampled the step before) and samples the next token once the prompt is read.
// Steps are enqueued T2S_CHUNK at a time as one graph; between chunks the host reads how many utterances have stopped, one
// chunk behind, so the device never waits for it.
static void impl_t2s_decode(vtts_handle h, const int64_t* ids, const int64_t* lengths, int B, int64_t ids_ld, const float* bert,
                            const int64_t* prompts, const int64_t* prompt_lengths, int64_t prompts_ld, int top_k, float top_p,
                            float temperature, float penalty, int early_stop, int step_cap, const uint64_t* seeds, const float* q,
                            int64_t q_ld, int64_t* tokens, int64_t tokens_ld, int64_t* n_tokens, int64_t* idx, float* logits,
                            int64_t logits_ld) {
  const vtts_config& c = h->cfg;
  const int H = c.cv_hidden, F = c.cv_ffn, nh = c.cv_heads, dk = H / nh, NL = c.cv_layers, V = h->t2s_vocab;
  REQUIRE(B >= 1 && B <= 4096, VTTS_ERR_INVALID, "bad batch size");
  REQUIRE(ids && lengths && ids_ld >= 1, VTTS_ERR_INVALID, "ids, lengths and ids_ld >= 1 are required");
  REQUIRE(top_k >= 1, VTTS_ERR_INVALID, "top_k must be at least 1");
  REQUIRE(std::isfinite(top_p) && std::isfinite(temperature) && std::isfinite(penalty) && penalty > 0.f, VTTS_ERR_INVALID,
          "top_p, temperature and a positive repetition penalty must be finite");
  REQUIRE(early_stop >= -1, VTTS_ERR_INVALID, "early_stop_num must be -1 (none) or >= 0");
  REQUIRE(step_cap >= 1 && step_cap <= (1 << 20), VTTS_ERR_INVALID, "the step cap must be in [1, 2^20]");
  REQUIRE(q || seeds, VTTS_ERR_INVALID, "give per-utterance seeds or q");
  REQUIRE(!prompts == !prompt_lengths, VTTS_ERR_INVALID, "prompts and prompt_lengths go together");
  const int gen_max = early_stop < 0 ? step_cap : std::min(step_cap, early_stop + 1);
  REQUIRE(!q || q_ld >= gen_max, VTTS_ERR_INVALID, "q must hold a row for every step that can sample (q_ld >= the step limit)");
  REQUIRE(!logits || logits_ld >= 1, VTTS_ERR_INVALID, "logits_ld must be >= 1");
  std::vector<int> T(B), P(B, 0), Lr(B), off(B), init(4 * (size_t)B), poff(B);
  long tot = 0, kvn = 0, ytot = 0, ptot = 0;
  int maxT = 0, maxKv = 0;
  for (int b = 0; b < B; ++b) {
    REQUIRE(lengths[b] >= 1 && lengths[b] <= ids_ld, VTTS_ERR_INVALID, "lengths must be in [1, ids_ld]");
    REQUIRE(lengths[b] <= h->t2s_npos, VTTS_ERR_INVALID, "a text is longer than the position table");
    T[b] = (int)lengths[b];
    for (int t = 0; t < T[b]; ++t) {
      const int64_t v = ids[(size_t)b * ids_ld + t];
      REQUIRE(v >= 0 && v < h->t2s_text_vocab, VTTS_ERR_INVALID, "a phone id is outside the text embedding table");
    }
    if (prompts) {
      REQUIRE(prompt_lengths[b] >= 0 && prompt_lengths[b] <= prompts_ld, VTTS_ERR_INVALID, "prompt_lengths must be in [0, prompts_ld]");
      P[b] = (int)prompt_lengths[b];
      for (int t = 0; t < P[b]; ++t) {
        const int64_t v = prompts[(size_t)b * prompts_ld + t];
        REQUIRE(v >= 0 && v < V - 1, VTTS_ERR_INVALID, "a prompt token is outside [0, EOS)");
      }
    }
    REQUIRE((long)P[b] + gen_max <= h->t2s_npos, VTTS_ERR_INVALID, "prompt plus the step limit is longer than the position table");
    REQUIRE(!tokens || tokens_ld >= (long)P[b] + gen_max, VTTS_ERR_CAPACITY, "tokens_ld is below a prompt length plus the step limit");
    off[b] = (int)tot;
    Lr[b] = T[b] + P[b];                             // prefill rows: the text, then the prompt
    tot += (Lr[b] + 7) / 8 * 8;
    const int kv = T[b] + P[b] + gen_max;
    init[4 * b] = T[b]; init[4 * b + 1] = P[b]; init[4 * b + 2] = (int)kvn; init[4 * b + 3] = (int)ytot;
    poff[b] = (int)ptot;
    kvn += kv; ytot += P[b] + gen_max; ptot += P[b];
    REQUIRE(tot < (1L << 24) && kvn < (1L << 28), VTTS_ERR_INVALID, "the batch holds too many rows for one call");
    maxT = std::max(maxT, Lr[b]); maxKv = std::max(maxKv, kv);
  }
  h->B = B;
  // staged: [T + P B][off B][init 4B][poff B][prefill ids tot][prompts ptot], the sampling scalars, the seeds and the BERT rows
  const size_t nint = 7 * (size_t)B + tot + ptot, nb = (size_t)tot * vtts_engine::T2S_BERT;
  vtts_engine::Staging& st = h->stg[vtts_engine::STG_T2S];
  st.begin();
  st.add(h->d_t2s_i, nint);
  st.add(h->d_t2s_prm, 1);
  st.add(h->d_t2s_seed, (size_t)B);
  if (bert) st.add(h->d_t2s_bert, nb);
  st.commit();
  int* pi = st.host(h->d_t2s_i);
  memcpy(pi, Lr.data(), B * sizeof(int));
  memcpy(pi + B, off.data(), B * sizeof(int));
  memcpy(pi + 2 * B, init.data(), 4 * (size_t)B * sizeof(int));
  memcpy(pi + 6 * B, poff.data(), B * sizeof(int));
  std::fill(pi + 7 * B, pi + 7 * B + tot, 0);
  for (int b = 0; b < B; ++b) {
    for (int t = 0; t < T[b]; ++t) pi[7 * B + off[b] + t] = (int)ids[(size_t)b * ids_ld + t];
    for (int t = 0; t < P[b]; ++t)
      pi[7 * B + off[b] + T[b] + t] = pi[7 * B + tot + poff[b] + t] = (int)prompts[(size_t)b * prompts_ld + t];
  }
  *st.host(h->d_t2s_prm) = T2sPrm{top_p, temperature, penalty, top_k, early_stop, step_cap, q ? (int)q_ld : 0, logits ? (int)logits_ld : 0};
  unsigned long long* psd = st.host(h->d_t2s_seed);
  for (int b = 0; b < B; ++b) psd[b] = seeds ? (unsigned long long)seeds[b] : 0ull;
  if (bert) {
    float* hb = st.host(h->d_t2s_bert);
    std::fill(hb, hb + nb, 0.f);
    for (int b = 0; b < B; ++b)
      memcpy(hb + (size_t)off[b] * vtts_engine::T2S_BERT, bert + (size_t)b * ids_ld * vtts_engine::T2S_BERT,
             (size_t)T[b] * vtts_engine::T2S_BERT * sizeof(float));
  }
  cudaStream_t s = h->stream;
  st.upload();
  const int* di = h->d_t2s_i.p;
  const T2sPrm* dprm = h->d_t2s_prm.p;
  const unsigned long long* dseed = h->d_t2s_seed.p;
  float* dq = nullptr;
  if (q) {
    dq = h->ensure(h->d_t2s_q, (size_t)B * q_ld * V);
    CK(cudaMemcpyAsync(dq, q, (size_t)B * q_ld * V * sizeof(float), cudaMemcpyHostToDevice, s));
  }
  float* draw = logits ? h->ensure(h->d_t2s_raw, (size_t)B * logits_ld * V) : nullptr;
  if (draw) CK(cudaMemsetAsync(draw, 0, (size_t)B * logits_ld * V * sizeof(float), s));
  const int* dlen = di;
  const int* doff = di + B;
  const int* dinit = di + 2 * B;

  // ---- prefill of the [text; prompt] rows under the prefix mask: one fixed launch shape per precision mode, so an
  //      utterance's rows do not depend on the batch
  const Tuning tn = h->t2s_tc ? h->tune.fixed_tc() : h->tune.fixed_ffma().fixed_attention();
  const Rows r{dlen, doff, B, maxT, std::vector<int>(B, maxT), Lr, tn};
  vtts_engine::PostLnWs w{h->ensure(h->d_t2s_x, tot * H), h->ensure(h->d_t2s_x1, tot * H), h->ensure(h->d_t2s_y, tot * H),
                          h->ensure(h->d_t2s_qkv, tot * 3 * H), h->ensure(h->d_t2s_ao, tot * H), h->ensure(h->d_t2s_ff, tot * F)};
  if (h->t2s_tc) {
    w.PX = h->planes(51, tot, 1, H); w.PQKV = h->planes(52, tot, 1, 3 * H);
    w.PAO = h->planes(53, tot, 1, H); w.PX1 = h->planes(54, tot, 1, H); w.PFF = h->planes(55, tot, 1, F);
  }
  float* kc = h->ensure(h->d_t2s_k, (size_t)NL * kvn * H);
  float* vc = h->ensure(h->d_t2s_v, (size_t)NL * kvn * H);
  const float* bp = nullptr;
  if (bert) {
    float* dbp = h->ensure(h->d_t2s_bp, (size_t)tot * H);
    h->launch_conv({mk(h->t2s_bp, h->d_t2s_bert.p, vtts_engine::T2S_BERT, 0, dbp, H, 0, 1, 0)}, 1, r);
    bp = dbp;
  }
  h->klaunch(t2s_prefill_embed_kernel, dim3(maxT, B), dim3(128), (size_t)0, (const int*)(di + 7 * B), h->t2s_temb, h->t2s_aemb, bp,
             h->t2s_bp.b, h->t2s_pe, h->t2s_alpha[0], h->t2s_alpha[1], H, w.xa, dlen, doff, dinit,
             h->t2s_tc ? w.PX.hi : (__nv_bfloat16*)nullptr, h->t2s_tc ? w.PX.lo : (__nv_bfloat16*)nullptr);
  CK(cudaGetLastError());
  ++h->launches;
  const std::function<void(int)> store = [&](int l) {
    h->klaunch(t2s_kv_store_kernel, dim3(maxT, B), dim3(128), (size_t)0, (const float*)w.QKV, H, kc + (size_t)l * kvn * H,
               vc + (size_t)l * kvn * H, dlen, doff, dinit);
    CK(cudaGetLastError());
    ++h->launches;
  };
  float* pre = h->ensure(h->d_t2s_pre, (size_t)tot * H);
  h->post_ln_layers(h->t2s_enc, h->t2s_tc, H, F, c.cv_ln_eps, w, pre, doff, r, true, &store, dinit);

  // ---- decode state
  const int rt = (B + T2S_RB - 1) / T2S_RB, nw = (V + 31) / 32;
  const int nsplit = ((maxKv + T2S_KS - 1) / T2S_KS + 7) / 8 * 8;
  int* dst = h->ensure(h->d_t2s_st, (size_t)B * T2S_ST + 1);
  int* nstop = dst + (size_t)B * T2S_ST;
  int* dy = h->ensure(h->d_t2s_tok, (size_t)ytot);
  unsigned* seen = h->ensure(h->d_t2s_seen, (size_t)B * nw);
  float* dec = h->ensure(h->d_t2s_dec, (size_t)B * (6 * H + F + V));
  float *dx = dec, *dqv = dx + (size_t)B * H, *y1 = dqv + (size_t)B * H, *xm = y1 + (size_t)B * H, *y2 = xm + (size_t)B * H,
        *hx = y2 + (size_t)B * H, *ff = hx + (size_t)B * H, *lg = ff + (size_t)B * F;
  float* part = h->ensure(h->d_t2s_part, (size_t)B * nh * nsplit * (dk + 2));
  CK(cudaMemsetAsync(nstop, 0, sizeof(int), s));
  h->klaunch(t2s_init_kernel, dim3(B), dim3(256), (size_t)0, dinit, (const int*)(di + 7 * B + tot), (const int*)(di + 6 * B), (const float*)pre,
             doff, H, V, dst, dy, seen, hx);
  CK(cudaGetLastError());
  ++h->launches;
  std::vector<T2sLayer> Ls(NL);
  for (int l = 0; l < NL; ++l) {
    const EncLayerW& E = h->t2s_enc[l];
    Ls[l] = T2sLayer{E.qkv.w, E.qkv.b, E.o.w, E.o.b, E.ffn1.w, E.ffn1.b, E.ffn2.w, E.ffn2.b, E.ln1.g, E.ln1.b, E.ln2.g, E.ln2.b,
                     E.qkv.ldw, E.o.ldw, E.ffn1.ldw, E.ffn2.ldw, c.cv_ln_eps, kc + (size_t)l * kvn * H, vc + (size_t)l * kvn * H};
  }
  const float scale = (float)std::sqrt(1.0 / dk);
  auto step = [&] {
    for (int l = 0; l < NL; ++l) {
      const T2sLayer& L = Ls[l];
      h->klaunch(t2s_qkv_kernel, dim3((3 * H + T2S_COLS - 1) / T2S_COLS, rt), dim3(32 * T2S_WARPS), T2S_GEMV_SMEM(H), L,
                 l ? Ls[l - 1].ln2g : (const float*)nullptr, l ? Ls[l - 1].ln2b : (const float*)nullptr, h->t2s_aemb, h->t2s_pe,
                 h->t2s_alpha[1], (const int*)dy, (const float*)y2, dx, dqv, (const int*)dst, B, H);
      h->klaunch(t2s_attn_kernel, dim3(nsplit, nh, B), dim3(32), (size_t)0, (const float*)dqv, (const float*)L.kc, (const float*)L.vc, part,
                 (const int*)dst, H, dk, scale, nsplit);
      h->klaunch(t2s_o_kernel, dim3((H + T2S_COLS - 1) / T2S_COLS, rt), dim3(32 * T2S_WARPS), T2S_GEMV_SMEM(H), L, (const float*)part,
                 (const float*)dx, y1, (const int*)dst, B, H, dk, nsplit);
      h->klaunch(t2s_ffn1_kernel, dim3((F + T2S_COLS - 1) / T2S_COLS, rt), dim3(32 * T2S_WARPS), T2S_GEMV_SMEM(H), L, (const float*)y1, xm,
                 ff, (const int*)dst, B, H, F);
      h->klaunch(t2s_ffn2_kernel, dim3((H + T2S_COLS - 1) / T2S_COLS, rt), dim3(32 * T2S_WARPS), T2S_GEMV_SMEM(F), L, (const float*)ff,
                 (const float*)xm, y2, (const int*)dst, B, H, F);
    }
    h->klaunch(t2s_logits_kernel, dim3((V + T2S_COLS - 1) / T2S_COLS, rt), dim3(32 * T2S_WARPS), T2S_GEMV_SMEM(H), h->t2s_pred.w,
               h->t2s_pred.ldw, Ls[NL - 1].ln2g, Ls[NL - 1].ln2b, c.cv_ln_eps, (const float*)y2, (const float*)hx, lg, (const int*)dst, B,
               H, V);
    h->klaunch(t2s_sample_kernel, dim3(B), dim3(T2S_SAMPLE_THREADS), (size_t)0, (const float*)lg, (const T2sPrm*)dprm,
               (const unsigned long long*)dseed, (const float*)dq, draw, dst, dy, seen, nstop, V);
    CK(cudaGetLastError());
    h->launches += 5 * (uint64_t)NL + 2;
  };
  // ---- readbacks, sized before the chunks' graphs capture (growth retires them): the stop count behind the state rows, one
  //      staging per chunk in flight; then the state rows and the tokens
  vtts_engine::Staging* stop = &h->stg[vtts_engine::STG_T2S_STOP0];
  for (int k = 0; k < 2; ++k) {
    stop[k].begin();
    stop[k].add(h->d_t2s_st, 1, (size_t)B * T2S_ST);
    stop[k].commit();
  }
  vtts_engine::Staging& out = h->stg[vtts_engine::STG_OUT];
  out.begin();
  out.add(h->d_t2s_st, (size_t)B * T2S_ST);
  out.add(h->d_t2s_tok, (size_t)ytot);
  out.commit();
  // ---- decode loop: every utterance has stopped after gen_max steps at the latest
  const long bound = gen_max;
  for (long it = 0, chunk = 0;; ++chunk) {
    h->run_graphed({vtts_engine::TAG_T2S, B, nsplit, kvn, ytot, q ? q_ld : -1, logits ? logits_ld : -1},
                   [&] { for (int k = 0; k < vtts_engine::T2S_CHUNK; ++k) step(); });
    stop[chunk & 1].download();
    CK(cudaEventRecord(h->ev[chunk & 1], s));
    it += vtts_engine::T2S_CHUNK;
    if (it >= bound) break;
    if (chunk >= 1) {
      CK(cudaEventSynchronize(h->ev[(chunk - 1) & 1]));
      if (*stop[(chunk - 1) & 1].host(h->d_t2s_st) >= B) break;
    }
  }
  // ---- read back (the caller's logits, up to B * logits_ld * V floats, straight to its memory, as q comes from it)
  if (logits) CK(cudaMemcpyAsync(logits, draw, (size_t)B * logits_ld * V * sizeof(float), cudaMemcpyDeviceToHost, s));
  out.download_and_wait();
  const int *sth = out.host(h->d_t2s_st), *yh = out.host(h->d_t2s_tok);
  for (int b = 0; b < B; ++b) {
    const int* sb = sth + (size_t)b * T2S_ST;
    REQUIRE(sb[ST_STOP] == 1, VTTS_ERR_STATE, "an utterance did not stop within its step limit");
    const int gen = sb[ST_GEN], n = P[b] + gen - 1;          // y[:, :-1]: the last appended token is dropped
    if (n_tokens) n_tokens[b] = n;
    if (idx) idx[b] = P[b] > 0 ? gen - 2 : 0;
    if (tokens)
      for (int i = 0; i < n; ++i) tokens[(size_t)b * tokens_ld + i] = yh[(size_t)init[4 * b + 3] + i];
  }
}

// QuickVC conversion through host buffers: from content units (vtts_quickvc_convert, wav null) or from source waveforms through
// ContentVec (vtts_quickvc_convert_wav, units null; in_ld is then wav_ld).
static void impl_quickvc_convert(vtts_handle h, const float* units, const float* wav, const int64_t* lengths, int B, int64_t in_ld,
                                 const float* g, float noise_scale, const float* noise, int noise_ld, uint64_t seed, float* out_wav,
                                 int64_t out_ld, int64_t* out_frames) {
  const vtts_config& c = h->cfg;
  const int64_t units_ld = in_ld;
  REQUIRE(h->has_encp, VTTS_ERR_INVALID, "the weight blob holds only the speaker encoder: conversion needs a model packed by "
          "weights.pack_quickvc from a whole QuickVC checkpoint (enc_p, flow, dec)");
  if (wav) require_contentvec(h, B);
  REQUIRE(B >= 1 && B <= 16384, VTTS_ERR_INVALID, "bad batch size");
  REQUIRE(in_ld >= 1 && (wav || units_ld < (1LL << 24)), VTTS_ERR_INVALID, wav ? "bad wav_ld" : "bad units_ld");
  REQUIRE(g != nullptr, VTTS_ERR_INVALID, "g (the target's speaker embedding, vtts_speaker_embedding) is required");
  std::vector<int> frames(B);
  if (wav) {
    REQUIRE(c.cv_hidden == vtts_engine::QV_UNITS, VTTS_ERR_INVALID, "ContentVec's width differs from enc_p's unit channels");
    h->B = B;
    frames = h->cv_stage(wav, lengths, in_ld);
  } else {
    for (int b = 0; b < B; ++b) {
      REQUIRE(lengths[b] >= 1 && lengths[b] <= units_ld, VTTS_ERR_INVALID, "unit_lengths must be in [1, units_ld]");
      frames[b] = (int)lengths[b];
    }
  }
  const int real_max = *std::max_element(frames.begin(), frames.end());
  REQUIRE((int64_t)real_max * h->hop <= out_ld, VTTS_ERR_CAPACITY, "out_ld is smaller than hop * max(unit_lengths)");
  REQUIRE(!noise || noise_ld >= real_max, VTTS_ERR_CAPACITY, "noise has fewer columns than max(unit_lengths)");
  h->B = B;
  h->have_durations = false;
  h->have_latent = false;
  h->pack_frames(frames);
  constexpr int U = vtts_engine::QV_UNITS;
  const int G = c.gin_channels;
  h->stage_clip_fields(units ? vtts_engine::IN_UNITS : vtts_engine::IN_NONE, noise != nullptr);
  vtts_engine::Staging& s = h->stg[vtts_engine::STG_CLIPS];
  memcpy(s.host(h->d_frm_len), frames.data(), B * sizeof(int));
  memcpy(s.host(h->d_frm_off), h->h_frm_off.data(), (B + 1) * sizeof(int));
  int* vi = s.host(h->d_vint);
  float* pin = units ? s.host(h->d_vin) : nullptr;
  for (int b = 0; b < B; ++b) {
    vi[b] = frames[b];
    vi[B + b] = b;                                      // cond_vc_kernel's row of g
    vi[2 * B + b] = 0;
    const int o = h->h_frm_off[b];
    if (units) {
      memcpy(pin + (size_t)o * U, units + (size_t)b * units_ld * U, (size_t)frames[b] * U * sizeof(float));
      const int gap_end = b + 1 < B ? h->h_frm_off[b + 1] : h->Tfrm;       // rows behind the clip: the gap, or the bucket's tail
      memset(pin + (size_t)(o + frames[b]) * U, 0, (size_t)(gap_end - o - frames[b]) * U * sizeof(float));
    }
  }
  memcpy(s.host(h->d_qg), g, (size_t)B * G * sizeof(float));
  if (noise) h->stage_noise(s.host(h->d_vnoise), noise, noise_ld, frames);
  vtts_engine::put_scalars(s.host(h->d_vprm), 16, &noise_scale, 1, seed);
  if (wav)
    h->run_graphed({vtts_engine::TAG_QUICKVC_WAV, B, h->maxFrm, h->Tfrm, noise ? 1 : 0, h->cvp.maxS, h->cvp.tot0},
                   [&] { h->quickvc_enqueue(noise != nullptr, true); });
  else
    h->run_graphed({vtts_engine::TAG_QUICKVC, B, h->maxFrm, h->Tfrm, noise ? 1 : 0}, [&] { h->quickvc_enqueue(noise != nullptr); });
  read_clips(read_back(h, h->d_wav, (size_t)h->real_Tfrm * h->hop, (size_t)h->Tfrm * h->hop), h->h_frm_off.data(), frames, h->hop,
             out_wav, out_ld);
  for (int b = 0; b < B; ++b) {
    std::fill(out_wav + (size_t)b * out_ld + (size_t)frames[b] * h->hop, out_wav + (size_t)(b + 1) * out_ld, 0.f);
    out_frames[b] = frames[b];
  }
}

// t_span = 1 - cos(linspace(0, 1, n + 1) pi / 2) and the Euler loop's t and dt into prm[16 ..], in the reference's fp32 steps
// (flow_matching.py:54-55,87-98: t accumulates, dt is the distance from it to the next knot)
static void st_schedule(float* prm, int n) {
  std::vector<float> span(n + 1);
  const float step = 1.f / (float)n;
  for (int i = 0; i <= n; ++i) {
    const float lin = i < (n + 1) / 2 ? step * (float)i : 1.f - step * (float)(n - i);
    const float a = (lin * 0.5f) * (float)M_PI;
    span[i] = 1.f - (float)std::cos((double)a);
  }
  float t = span[0], dt = span[1] - span[0];
  for (int k = 0; k < n; ++k) {
    prm[16 + k] = t;
    prm[16 + VTTS_CFM_MAX_STEPS + k] = dt;
    t = t + dt;
    if (k + 1 < n) dt = span[k + 2] - t;
  }
}

// The flow-matching plan of a call and its staged inputs: d_sti [len NS][off NS][sid NS][extent NS], where sequence q < B is
// utterance q's conditional branch and B + q its unconditional one (rows packed by extent); d_stf prm[16] | t[64] | dt[64] |
// speaker rows [B][G] (rows); the mu rows [Tfrm][MC] packed as the engine's rows (vtts_cfm_decode; text-to-mel expands them
// on the device); the noise rows [Tfrm][NC] (noise).  The caller fills the speaker, mu and noise rows.
static void st_plan(vtts_handle h, int B, const std::vector<int>& frames, const std::vector<int>& extents, const int64_t* sid, int n,
                    float temperature, float s, bool noise, bool rows, bool text, bool prior, int denormalise, uint64_t seed) {
  h->pack_frames(extents);
  vtts_engine::StPlan& P = h->stp;
  P.guided = s > 0.f;
  P.NS = P.guided ? 2 * B : B;
  P.steps = n;
  P.noise = noise;
  P.rows = rows;
  P.text = text;
  P.prior = prior;
  P.Ttot = P.guided ? 2 * h->Tfrm + SEQ_GAP : h->Tfrm;
  REQUIRE((int64_t)P.Ttot * 3 * h->cfg.st_filter < (int64_t)INT32_MAX, VTTS_ERR_INVALID, "the batch holds too many frames for one call");
  const int NS = P.NS;
  const vtts_config& c = h->cfg;
  vtts_engine::Staging& st = h->stg[vtts_engine::STG_ST_MEL];
  st.begin();
  st.add(h->d_sti, 4 * (size_t)NS);
  st.add(h->d_stf, vtts_engine::ST_PRM + (rows ? (size_t)B * c.st_spk_dim : 0));
  if (!text) st.add(h->d_stmu, (size_t)h->Tfrm * c.st_cond);
  if (noise) st.add(h->d_stnoise, (size_t)h->Tfrm * c.st_noise);
  st.commit();
  int* pi = st.host(h->d_sti);
  for (int q = 0; q < NS; ++q) {
    const int b = q < B ? q : q - B;
    pi[q] = frames[b];
    pi[NS + q] = h->h_frm_off[b] + (q < B ? 0 : h->Tfrm + SEQ_GAP);
    pi[2 * NS + q] = q < B ? (sid ? (int)sid[b] : 0) : -1;
    pi[3 * NS + q] = extents[b];
  }
  const float sc[3] = {temperature, s, denormalise ? 1.f : 0.f};
  float* prm = st.host(h->d_stf);
  vtts_engine::put_scalars(prm, vtts_engine::ST_PRM, sc, 3, seed);
  st_schedule(prm, n);
}

static void st_check_sampling(int n, float temperature, float s) {
  REQUIRE(n >= 1 && n <= VTTS_CFM_MAX_STEPS, VTTS_ERR_INVALID, "n_timesteps must be in [1, " + std::to_string(VTTS_CFM_MAX_STEPS) + "]");
  REQUIRE(std::isfinite(temperature), VTTS_ERR_INVALID, "temperature must be finite");
  REQUIRE(std::isfinite(s) && s >= 0.f, VTTS_ERR_INVALID, "guidance_scale must be finite and >= 0");
}

// StableTTS flow-matching decoder through host buffers (vtts_cfm_decode).
static void impl_cfm_decode(vtts_handle h, const float* mu, const int64_t* lengths, int B, int64_t mu_ld, const int64_t* sid,
                            const float* spk_rows, int n, float temperature, float s, const float* noise, int64_t noise_ld, uint64_t seed,
                            float* mel_out, int64_t mel_ld, int denormalise) {
  const vtts_config& c = h->cfg;
  REQUIRE(B >= 1 && B <= 8192 && mu_ld >= 1 && mu_ld < (1LL << 24), VTTS_ERR_INVALID, "bad batch size / mu_ld");
  st_check_sampling(n, temperature, s);
  REQUIRE(sid || spk_rows, VTTS_ERR_INVALID, "a speaker is required: sid or spk_rows");
  std::vector<int> frames(B);
  for (int b = 0; b < B; ++b) {
    REQUIRE(lengths[b] >= 1 && lengths[b] <= mu_ld, VTTS_ERR_INVALID, "lengths must be in [1, mu_ld]");
    REQUIRE(spk_rows || (sid[b] >= 0 && sid[b] < c.st_n_spks), VTTS_ERR_INVALID, "speaker id out of range [0, n_spks)");
    frames[b] = (int)lengths[b];
  }
  const int real_max = *std::max_element(frames.begin(), frames.end());
  REQUIRE(mel_ld >= real_max, VTTS_ERR_CAPACITY, "mel_ld is smaller than the longest utterance");
  REQUIRE(!noise || noise_ld >= real_max, VTTS_ERR_CAPACITY, "noise has fewer frames than the longest utterance");
  h->B = B;
  h->have_durations = false;
  h->have_latent = false;
  const int NC = c.st_noise, MC = c.st_cond, G = c.st_spk_dim;
  st_plan(h, B, frames, frames, sid, n, temperature, s, noise != nullptr, spk_rows != nullptr, false, false, denormalise, seed);
  const vtts_engine::StPlan& P = h->stp;
  vtts_engine::Staging& st = h->stg[vtts_engine::STG_ST_MEL];
  if (spk_rows) memcpy(st.host(h->d_stf) + vtts_engine::ST_PRM, spk_rows, (size_t)B * G * sizeof(float));
  float* pmu = st.host(h->d_stmu);
  float* pn = noise ? st.host(h->d_stnoise) : nullptr;
  for (int b = 0; b < B; ++b) {
    const size_t o = (size_t)h->h_frm_off[b];
    memcpy(pmu + o * MC, mu + (size_t)b * mu_ld * MC, (size_t)frames[b] * MC * sizeof(float));
    if (noise) memcpy(pn + o * NC, noise + (size_t)b * noise_ld * NC, (size_t)frames[b] * NC * sizeof(float));
  }
  h->run_graphed({vtts_engine::TAG_CFM, B, h->maxFrm, h->Tfrm, n, P.guided ? 1 : 0, P.noise ? 1 : 0, P.rows ? 1 : 0}, [&] { h->st_enqueue(); });
  read_clips(read_back(h, h->d_stmel, (size_t)h->real_Tfrm * NC, (size_t)h->Tfrm * NC), h->h_frm_off.data(), frames, NC, mel_out,
             mel_ld * NC);
}

// StableTTS text-to-mel through host buffers (vtts_stabletts_synthesise): the text phase, one wait for the frame counts, the
// mel phase.
static void impl_stabletts_synthesise(vtts_handle h, const int64_t* ids, const int64_t* id_lengths, int B, int64_t t_max, const float* bert,
                                      const float* pause, const int64_t* sid, int n, float temperature, float length_scale, float s,
                                      const float* noise, int64_t noise_ld, uint64_t seed, float* mel_out, int64_t mel_ld, int64_t* mel_lengths,
                                      int32_t* durations, float* prior_out, int denormalise, float* wav = nullptr, int64_t wav_ld = 0,
                                      int64_t* wav_lengths = nullptr, const int64_t* pieces = nullptr, const int64_t* piece_lengths = nullptr,
                                      int64_t pieces_ld = 0, const int32_t* bert_rows = nullptr) {
  const vtts_config& c = h->cfg;
  REQUIRE(!wav || h->has_voc, VTTS_ERR_INVALID, "the weight blob has no vocoder (StableTTS(..., vocoder=...) / weights.pack_hifigan)");
  REQUIRE(h->st_text, VTTS_ERR_INVALID, "the weight blob holds the flow-matching decoder only (weights.pack_stabletts_cfm): text-to-mel needs the "
                                         "text encoder of weights.pack_stabletts");
  REQUIRE(!prior_out || h->st_prior, VTTS_ERR_INVALID, "the weight blob has no mel encoder (encoder.encoder.*, which an exported graph "
                                                          "drops): the prior (encoder_outputs) cannot be computed");
  REQUIRE(B >= 1 && B <= 8192 && t_max >= 1 && t_max <= VTTS_ST_MAX_TOKENS, VTTS_ERR_INVALID, "bad batch size / t_max");
  st_check_sampling(n, temperature, s);
  REQUIRE(std::isfinite(length_scale) && length_scale > 0.f && length_scale <= 100.f, VTTS_ERR_INVALID, "length_scale must be in (0, 100]");
  const int S = c.st_streams, BD = c.st_bert_dim, NC = c.st_noise;
  for (int b = 0; b < B; ++b) {
    REQUIRE(id_lengths[b] >= 1 && id_lengths[b] <= t_max, VTTS_ERR_INVALID, "id_lengths must be in [1, t_max]");
    REQUIRE(sid[b] >= 0 && sid[b] < c.st_n_spks, VTTS_ERR_INVALID, "speaker id out of range [0, n_spks)");
    for (int q = 0; q < S; ++q)
      for (int64_t i = 0; i < id_lengths[b]; ++i) {
        const int64_t v = ids[((size_t)b * S + q) * t_max + i];
        REQUIRE(v >= 0 && v < c.st_n_vocab, VTTS_ERR_INVALID, "token id out of range [0, n_vocab)");
      }
    if (pause)
      for (int64_t i = 0; i < id_lengths[b]; ++i) {
        const float v = pause[(size_t)b * t_max + i];
        REQUIRE(v >= 0.f && v <= (float)VTTS_ST_MAX_TOKEN_FRAMES, VTTS_ERR_INVALID, "pause durations must be in [0, VTTS_ST_MAX_TOKEN_FRAMES]");
      }
  }
  if (pieces) {
    REQUIRE(h->has_bert, VTTS_ERR_INVALID, "the weight blob has no BERT (bt.*): build the engine with StableTTS(..., bert=...)");
    REQUIRE(BD == c.cv_hidden, VTTS_ERR_INVALID, "bert_dim differs from BERT's hidden width");
    REQUIRE(pieces_ld >= 1, VTTS_ERR_INVALID, "bad pieces_ld");
    for (int b = 0; b < B; ++b)
      for (int64_t i = 0; i < id_lengths[b]; ++i) {
        const int32_t v = bert_rows[(size_t)b * t_max + i];
        REQUIRE(v >= 0 && v < piece_lengths[b], VTTS_ERR_INVALID, "a BERT row is outside its sentence's word pieces [0, piece_lengths)");
      }
  }
  setup_lengths(h, id_lengths, B, (int)t_max);
  if (pieces) h->bt_stage(pieces, piece_lengths, pieces_ld);
  const int Ttok = h->Ttok;
  {
    // [tok len B][tok off B][sid B][ids streams x Ttok]; prm[16] | pause [Ttok]; the BERT rows [Ttok][bert_dim] (without
    // pieces), tokens packed as the engine's rows
    vtts_engine::Staging& st = h->stg[vtts_engine::STG_ST_TEXT];
    st.begin();
    st.add(h->d_stti, (size_t)3 * B + (size_t)S * Ttok);
    st.add(h->d_sttf, 16 + (size_t)Ttok);
    if (!pieces) st.add(h->d_stbert, (size_t)Ttok * BD);
    st.commit();
    int* pi = st.host(h->d_stti);
    float* prm = st.host(h->d_sttf);
    float* pp = prm + 16;
    memset(pi + 3 * B, 0, (size_t)S * Ttok * sizeof(int));
    std::fill(pp, pp + Ttok, 0.f);
    vtts_engine::put_scalars(prm, 16, &length_scale, 1, seed);
    for (int b = 0; b < B; ++b) {
      const int len = h->h_tok_len[b], o = h->h_tok_off[b];
      pi[b] = len;
      pi[B + b] = o;
      pi[2 * B + b] = (int)sid[b];
      for (int q = 0; q < S; ++q)
        for (int i = 0; i < len; ++i) pi[3 * B + (size_t)q * Ttok + o + i] = (int)ids[((size_t)b * S + q) * t_max + i];
      if (pause) memcpy(pp + o, pause + (size_t)b * t_max, (size_t)len * sizeof(float));
      if (bert) memcpy(st.host(h->d_stbert) + (size_t)o * BD, bert + (size_t)b * t_max * BD, (size_t)len * BD * sizeof(float));
    }
  }
  const bool prior = prior_out != nullptr;
  vtts_engine::Staging& sd = h->stg[vtts_engine::STG_ST_DURATIONS];     // (downloaded inside the text phase's graph)
  sd.begin();
  sd.add(h->d_sttd, 2 * (size_t)Ttok + B);
  sd.commit();
  if (pieces) {
    vtts_engine::Staging& sg = h->stg[vtts_engine::STG_ST_PIECES];
    sg.begin();
    sg.add(h->d_stg, 2 * (size_t)B + Ttok);
    sg.commit();
    int* g = sg.host(h->d_stg);
    memcpy(g, h->h_tok_len.data(), B * sizeof(int));
    memcpy(g + B, h->h_tok_off.data(), B * sizeof(int));
    std::fill(g + 2 * B, g + 2 * B + Ttok, 0);
    for (int b = 0; b < B; ++b)
      for (int i = 0; i < h->h_tok_len[b]; ++i) g[2 * B + h->h_tok_off[b] + i] = h->btp.off[b] + bert_rows[(size_t)b * t_max + i];
    h->run_graphed({vtts_engine::TAG_ST_TEXT_PIECES, B, h->maxTok, Ttok, prior ? 1 : 0, h->btp.maxL, h->btp.tot}, [&] {
      h->stt_bert_enqueue();
      h->stt_enqueue(prior);
    });
  } else {
    h->run_graphed({vtts_engine::TAG_ST_TEXT, B, h->maxTok, Ttok, prior ? 1 : 0}, [&] { h->stt_enqueue(prior); });
  }
  CK(cudaStreamSynchronize(h->stream));            // the one wait of the path: the frame counts size the mel phase
  const int* sttd = sd.host(h->d_sttd);
  std::vector<int> frames(B), extents(B);
  int64_t total = 0;
  for (int b = 0; b < B; ++b) {
    frames[b] = sttd[2 * (size_t)Ttok + b];
    extents[b] = (frames[b] + 3) / 4 * 4;
    mel_lengths[b] = frames[b];
    total += extents[b];
    if (durations) {
      std::fill(durations + (size_t)b * t_max, durations + (size_t)(b + 1) * t_max, 0);
      memcpy(durations + (size_t)b * t_max, sttd + h->h_tok_off[b], (size_t)h->h_tok_len[b] * sizeof(int));
    }
  }
  REQUIRE(total < (1LL << 24), VTTS_ERR_INVALID, "the batch expands to too many frames for one call");
  const int real_max = *std::max_element(frames.begin(), frames.end()), ext_max = (real_max + 3) / 4 * 4;
  REQUIRE(!mel_out || mel_ld >= real_max, VTTS_ERR_CAPACITY, "mel_ld is smaller than the longest utterance (mel_lengths holds the frame counts)");
  REQUIRE(!wav || wav_ld >= (int64_t)real_max * h->hop, VTTS_ERR_CAPACITY,
          "wav_ld is smaller than the longest utterance times the hop (mel_lengths holds the frame counts)");
  REQUIRE(!noise || noise_ld >= ext_max, VTTS_ERR_CAPACITY, "noise has fewer frames than the longest utterance padded to a multiple of 4 "
                                                            "(mel_lengths holds the frame counts)");
  st_plan(h, B, frames, extents, sid, n, temperature, s, noise != nullptr, false, true, prior, denormalise, seed);
  const vtts_engine::StPlan& P = h->stp;
  if (noise)
    for (int b = 0; b < B; ++b)
      memcpy(h->stg[vtts_engine::STG_ST_MEL].host(h->d_stnoise) + (size_t)h->h_frm_off[b] * NC, noise + (size_t)b * noise_ld * NC,
             (size_t)extents[b] * NC * sizeof(float));
  // the vocoder reads the conditional sequences' rows: lens and offsets are the first B of the phase's [len NS][off NS] table
  h->run_graphed({vtts_engine::TAG_ST_MEL, B, h->maxFrm, h->Tfrm, n, P.guided ? 1 : 0, P.noise ? 1 : 0, prior ? 1 : 0, h->maxTok, Ttok, wav ? 1 : 0},
                 [&] {
                   h->st_enqueue();
                   if (wav) {
                     const int *lens = h->d_sti.p, *offs = lens + P.NS;
                     float* in = h->ensure(h->d_hgmel, (size_t)h->Tfrm * NC);
                     h->klaunch(hg_mel_in_kernel, dim3(h->maxFrm, B), dim3(128), (size_t)0, (const float*)h->d_stmel.p, NC, (const float*)h->d_stf.p,
                                h->st_mel_mean, h->st_mel_std, in, lens, offs);
                     CK(cudaGetLastError());
                     ++h->launches;
                     h->voc_enqueue(in, lens, offs);
                   }
                 });
  // d_stmel holds the mel plane [Tfrm][NC], then with `prior` the prior's
  const size_t plane = (size_t)h->Tfrm * NC;
  vtts_engine::Staging& so = h->stg[vtts_engine::STG_OUT];
  so.begin();
  if (mel_out || prior) so.add(h->d_stmel, (prior ? plane : 0) + (size_t)h->real_Tfrm * NC, 0, 2 * plane);
  if (wav) so.add(h->d_wav, (size_t)h->real_Tfrm * h->hop, 0, (size_t)h->Tfrm * h->hop);
  so.commit();
  so.download_and_wait();
  for (int b = 0; b < B; ++b) {
    const size_t o = (size_t)h->h_frm_off[b] * NC, nb = (size_t)frames[b] * NC * sizeof(float);
    if (mel_out) memcpy(mel_out + (size_t)b * mel_ld * NC, so.host(h->d_stmel) + o, nb);
    if (prior) memcpy(prior_out + (size_t)b * mel_ld * NC, so.host(h->d_stmel) + plane + o, nb);
    if (wav) {
      memcpy(wav + (size_t)b * wav_ld, so.host(h->d_wav) + (size_t)h->h_frm_off[b] * h->hop, (size_t)frames[b] * h->hop * sizeof(float));
      wav_lengths[b] = (int64_t)frames[b] * h->hop;
    }
  }
}

static void require_vocoder(vtts_handle h) {
  REQUIRE(h->has_voc, VTTS_ERR_INVALID, "the weight blob has no vocoder (StableTTS(..., vocoder=...) / weights.pack_hifigan)");
}

// Rows of the largest buffer the vocoder allocates for a packed batch of `rows` frames must stay below 2^31 values.
static void voc_check_rows(vtts_handle h, int64_t rows) {
  const vtts_config& c = h->cfg;
  int64_t rm = 1, ch = c.upsample_initial_channel, most = rows * ch;
  for (int i = 0; i < c.n_upsamples; ++i) { rm *= c.upsample_rates[i]; ch /= 2; most = std::max(most, rows * rm * ch); }
  REQUIRE(most < (int64_t)INT32_MAX, VTTS_ERR_INVALID, "the batch holds too many frames for one vocoder call");
}

// StableTTS vocoder through host buffers (vtts_hifigan_vocode): one graphed enqueue per (batch, frame bucket).
static void impl_hifigan_vocode(vtts_handle h, const float* mel, const int64_t* mel_lengths, int B, int64_t mel_ld, float* wav, int64_t wav_ld,
                                int64_t* wav_lengths) {
  const vtts_config& c = h->cfg;
  require_vocoder(h);
  REQUIRE(B >= 1 && B <= 8192 && mel_ld >= 1 && mel_ld < (1LL << 24), VTTS_ERR_INVALID, "bad batch size / mel_ld");
  std::vector<int> frames(B);
  int64_t total = 0;
  for (int b = 0; b < B; ++b) {
    REQUIRE(mel_lengths[b] >= 1 && mel_lengths[b] <= mel_ld, VTTS_ERR_INVALID, "mel_lengths must be in [1, mel_ld]");
    frames[b] = (int)mel_lengths[b];
    total += frames[b] + SEQ_GAP;
  }
  voc_check_rows(h, total + 1024);
  const int real_max = *std::max_element(frames.begin(), frames.end());
  REQUIRE(wav_ld >= (int64_t)real_max * h->hop, VTTS_ERR_CAPACITY, "wav_ld is smaller than the longest utterance times the hop");
  const int NC = c.st_noise;
  h->B = B;
  h->have_durations = false;
  h->have_latent = false;
  h->pack_frames(frames);
  voc_check_rows(h, h->Tfrm);
  // staged: [len B][off B], then the mel rows [Tfrm][NC] packed as the engine's rows
  vtts_engine::Staging& st = h->stg[vtts_engine::STG_VOCODER];
  st.begin();
  st.add(h->d_hgi, 2 * (size_t)B);
  st.add(h->d_hgmel, (size_t)h->Tfrm * NC);
  st.commit();
  int* pi = st.host(h->d_hgi);
  float* pm = st.host(h->d_hgmel);
  for (int b = 0; b < B; ++b) {
    pi[b] = frames[b];
    pi[B + b] = h->h_frm_off[b];
    memcpy(pm + (size_t)h->h_frm_off[b] * NC, mel + (size_t)b * mel_ld * NC, (size_t)frames[b] * NC * sizeof(float));
  }
  h->run_graphed({vtts_engine::TAG_HIFIGAN, B, h->maxFrm, h->Tfrm}, [&] {
    int* di = h->ensure(h->d_hgi, 2 * (size_t)B);
    float* dm = h->ensure(h->d_hgmel, (size_t)h->Tfrm * NC);
    st.upload();
    h->voc_enqueue(dm, di, di + B);
  });
  read_clips(read_back(h, h->d_wav, (size_t)h->real_Tfrm * h->hop, (size_t)h->Tfrm * h->hop), h->h_frm_off.data(), frames, h->hop, wav,
             wav_ld);
  for (int b = 0; b < B; ++b) wav_lengths[b] = (int64_t)frames[b] * h->hop;
}

// I0 by its power series (the Kaiser window's; np.i0 within a few ulps for the beta 5 of resample_poly)
static double bessel_i0(double x) {
  double sum = 1.0, term = 1.0;
  for (int k = 1; k < 200 && term > 1e-18 * sum; ++k) {
    const double r = x / (2.0 * k);
    term *= r * r;
    sum += term;
  }
  return sum;
}

}  // namespace

// The low-pass of resample_poly for (up, down) (firwin(2 half + 1, 1 / max(up, down), window=("kaiser", 5.0)) * up, half =
// 10 max(up, down)) in float64, rounded to fp32 once, laid out per phase [up][K]: phase p holds h[p + up q], zeros past L.
const vtts_engine::RsTaps& vtts_engine::resample_taps(int up, int down) {
  RsTaps& r = rs_taps[{up, down}];
  if (r.taps.p) return r;
  const int M = std::max(up, down), half = 10 * M, L = 2 * half + 1, K = (L + up - 1) / up;
  std::vector<double> h(L);
  const double pi = 3.14159265358979323846, alpha = 0.5 * (L - 1), i0b = bessel_i0(5.0);
  double sum = 0.0;
  for (int i = 0; i < L; ++i) {
    const double n = (double)(i - half) / M, u = (i - alpha) / alpha;
    const double sinc = n == 0.0 ? 1.0 : std::sin(pi * n) / (pi * n);
    h[i] = sinc / M * (bessel_i0(5.0 * std::sqrt(std::max(0.0, 1.0 - u * u))) / i0b);
    sum += h[i];
  }
  std::vector<float> poly((size_t)up * K, 0.f);
  for (int i = 0; i < L; ++i) poly[(size_t)(i % up) * K + i / up] = (float)(h[i] / sum * up);
  Buf<float> buf;
  CK(buf.alloc(poly.size()));
  // On the engine's stream, so that the kernels enqueued behind it read the taps only after the copy has landed (the stream
  // is non-blocking: a cudaMemcpy on the legacy stream would not order them).  A pageable source is staged before the call
  // returns, so `poly` may go when it does.
  CK(cudaMemcpyAsync(buf.p, poly.data(), poly.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
  r.taps = std::move(buf);
  r.up = up; r.down = down; r.K = K;
  return r;
}

namespace {

// Resampling (and trimming) through host buffers (vtts_resample): the clips are packed as rows with SEQ_GAP between them
// into pinned staging with the row table, uploaded, resampled (equal rates: the uploaded rows are the output), the frame
// energies of the trim computed on the device and read back, the bounds picked on the host, then the kept rows read back.
static void impl_resample(vtts_handle h, const float* wav, const int64_t* lengths, int B, int64_t ld, int from_rate, int to_rate,
                          float trim_top_db, float* out, int64_t out_ld, int64_t* out_lengths, int64_t* trim_bounds) {
  REQUIRE(wav && lengths && out && out_lengths, VTTS_ERR_INVALID, "wav, lengths, out and out_lengths are required");
  REQUIRE(B >= 1 && B <= 16384, VTTS_ERR_INVALID, "bad batch size");
  REQUIRE(ld >= 1, VTTS_ERR_INVALID, "bad wav_ld");
  for (int r : {from_rate, to_rate})
    REQUIRE(r >= VTTS_RESAMPLE_MIN_RATE && r <= VTTS_RESAMPLE_MAX_RATE, VTTS_ERR_INVALID,
            "sample rates must lie in [" + std::to_string(VTTS_RESAMPLE_MIN_RATE) + ", " + std::to_string(VTTS_RESAMPLE_MAX_RATE) +
            "] Hz, not " + std::to_string(r));
  int a = from_rate, c = to_rate;
  while (c) { const int t = a % c; a = c; c = t; }
  const int up = to_rate / a, down = from_rate / a;
  const int64_t ntaps = 20LL * std::max(up, down) + 1;
  REQUIRE(ntaps <= VTTS_RESAMPLE_MAX_TAPS, VTTS_ERR_INVALID,
          "resampling " + std::to_string(from_rate) + " -> " + std::to_string(to_rate) + " Hz needs a filter of " +
          std::to_string(ntaps) + " taps, more than the " + std::to_string(VTTS_RESAMPLE_MAX_TAPS) + " this call supports");
  const bool same = up == down;
  std::vector<int> in_len(B), out_len(B), in_off, out_off, e_off(B + 1, 0);
  int64_t total = 0;
  for (int b = 0; b < B; ++b) {
    REQUIRE(lengths[b] >= 1 && lengths[b] <= ld, VTTS_ERR_INVALID, "wav_lengths must be in [1, wav_ld]");
    const int64_t n = ((int64_t)lengths[b] * up + down - 1) / down;
    REQUIRE(n <= out_ld, VTTS_ERR_CAPACITY, "out_ld is smaller than a resampled clip (ceil(len * to_rate / from_rate))");
    total += std::max<int64_t>(lengths[b], n) + SEQ_GAP;
    REQUIRE(total <= VTTS_RESAMPLE_MAX_BATCH_SAMPLES, VTTS_ERR_INVALID, "the batch holds too many samples for one call");
    in_len[b] = (int)lengths[b];
    out_len[b] = (int)n;
    e_off[b + 1] = e_off[b] + 1 + out_len[b] / RS_HOP;
  }
  vtts_engine::pack_rows(in_len, in_off);
  if (same) out_off = in_off;
  else vtts_engine::pack_rows(out_len, out_off);
  // staging: the row table, then the packed input rows
  vtts_engine::Staging& st = h->stg[vtts_engine::STG_RESAMPLE];
  st.begin();
  st.add(h->d_rsi, (size_t)5 * B);
  st.add(h->d_rsin, (size_t)in_off[B]);
  st.commit();
  int* tab = st.host(h->d_rsi);
  float* pin = st.host(h->d_rsin);
  for (int b = 0; b < B; ++b) {
    tab[b] = in_off[b]; tab[B + b] = in_len[b]; tab[2 * B + b] = out_off[b]; tab[3 * B + b] = out_len[b]; tab[4 * B + b] = e_off[b];
    memcpy(pin + in_off[b], wav + (size_t)b * ld, (size_t)in_len[b] * sizeof(float));
  }
  st.upload();
  const int* di = h->d_rsi.p;
  const float* din = h->d_rsin.p;
  const int max_out = *std::max_element(out_len.begin(), out_len.end());
  const float* y = din;
  if (!same) {
    const vtts_engine::RsTaps& rt = h->resample_taps(up, down);
    const int K = rt.K, half = 10 * std::max(up, down);
    int tile = RS_TILE_MAX;
    while (tile > 32 && rs_window(tile, up, down, K) > RS_WIN_MAX) tile /= 2;
    const int taps_smem = (int64_t)up * rs_taps_pitch(K) <= RS_TAPS_SMEM ? 1 : 0;
    const size_t smem = ((size_t)(taps_smem ? up * rs_taps_pitch(K) : 0) + rs_window(tile, up, down, K)) * sizeof(float);
    REQUIRE(smem <= 200 * 1024, VTTS_ERR_INVALID, "resampler window does not fit shared memory");
    CK(cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    float* dout = h->ensure(h->d_rsout, (size_t)out_off[B]);
    h->klaunch(resample_kernel, dim3((max_out + tile - 1) / tile, B), dim3(RS_THREADS), smem, (const float*)din, (const int*)di, B,
               (const float*)rt.taps.p, up, down, K, half, tile, taps_smem, dout);
    CK(cudaGetLastError());
    ++h->launches;
    y = dout;
  }
  std::vector<int> keep_off(out_off.begin(), out_off.begin() + B), keep_len = out_len;
  if (trim_top_db > 0.f) {
    const int max_nf = 1 + max_out / RS_HOP;
    double* de = h->ensure(h->d_rse, (size_t)e_off[B]);
    h->klaunch(frame_energy_kernel, dim3((max_nf + RS_FRAME_WARPS - 1) / RS_FRAME_WARPS, B), dim3(RS_FRAME_WARPS * 32), (size_t)0, y,
               (const int*)(di + 2 * B), B, de);
    CK(cudaGetLastError());
    ++h->launches;
    vtts_engine::Staging& se = h->stg[vtts_engine::STG_TRIM];
    se.begin();
    se.add(h->d_rse, (size_t)e_off[B]);
    se.commit();
    se.download_and_wait();
    const double* pe = se.host(h->d_rse);
    const double amin = 1e-10, thr = -(double)trim_top_db;
    for (int b = 0; b < B; ++b) {
      const double* e = pe + e_off[b];
      const int nf = e_off[b + 1] - e_off[b];
      double top = 0.0;
      for (int f = 0; f < nf; ++f) top = std::max(top, e[f] / RS_FRAME);
      REQUIRE(top > amin, VTTS_ERR_INVALID, "clip " + std::to_string(b) +
              " is silent throughout (every frame's mean square is at most 1e-10): trimming leaves nothing to keep");
      const double ref = 10.0 * std::log10(std::max(amin, top));
      int first = -1, last = -1;
      for (int f = 0; f < nf; ++f) {
        if (10.0 * std::log10(std::max(amin, e[f] / RS_FRAME)) - ref > thr) {
          if (first < 0) first = f;
          last = f;
        }
      }
      const int s0 = first * RS_HOP, s1 = std::min(out_len[b], (last + 1) * RS_HOP);
      keep_off[b] = out_off[b] + s0;
      keep_len[b] = s1 - s0;
      if (trim_bounds) { trim_bounds[2 * b] = s0; trim_bounds[2 * b + 1] = s1; }
    }
  } else if (trim_bounds) {
    for (int b = 0; b < B; ++b) { trim_bounds[2 * b] = 0; trim_bounds[2 * b + 1] = out_len[b]; }
  }
  // read back the packed span from the first kept sample to the last (with a trim: not the first clip's leading and the last
  // clip's trailing silence)
  const int lo = keep_off[0], hi = keep_off[B - 1] + keep_len[B - 1];
  for (int& o : keep_off) o -= lo;
  read_clips(read_back(h, same ? h->d_rsin : h->d_rsout, (size_t)(hi - lo), 0, (size_t)lo), keep_off.data(), keep_len, 1, out, out_ld);
  for (int b = 0; b < B; ++b) out_lengths[b] = keep_len[b];
}

static void impl_synthesize_dev(vtts_handle h, const float* d_noise_z, int z_ld, float* d_wav, int64_t wav_ld) {
  REQUIRE(h->have_durations, VTTS_ERR_STATE, "vtts_synthesize_dev called without vtts_durations_dev");
  REQUIRE((int64_t)h->real_maxFrm * h->hop <= wav_ld, VTTS_ERR_CAPACITY, "wav_ld is smaller than hop * max(y_lengths)");
  REQUIRE(!d_noise_z || z_ld >= h->real_maxFrm, VTTS_ERR_CAPACITY, "noise_z has fewer columns than max(y_lengths)");
  h->run_graphed({vtts_engine::TAG_PHASE2_DEV, h->B, h->maxFrm, h->Tfrm, z_ld, (long long)(uintptr_t)d_noise_z}, [&] { h->phase2(d_noise_z, z_ld, true); });
  for (int b = 0; b < h->B; ++b)
    CK(cudaMemcpyAsync(d_wav + (size_t)b * wav_ld, h->d_wav.p + (size_t)h->h_frm_off[b] * h->hop,
                       (size_t)h->h_frm_len[b] * h->hop * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaEventRecord(h->ev[7], h->stream));
  CK(cudaStreamSynchronize(h->stream));
  collect_timings(h);
  h->have_durations = false;
}

}  // namespace

extern "C" {

int vtts_create(const vtts_config* cfg, const float* blob, size_t blob_floats, const char* manifest, int blob_is_device,
                int device, vtts_handle* out) {
  if (!cfg || !blob || !manifest || !out) return VTTS_ERR_INVALID;
  *out = nullptr;
  vtts_engine* h = new vtts_engine();
  for (int k = 0; k < vtts_engine::STG_KINDS; ++k) { h->stg[k].e = h; h->stg[k].readback = k >= vtts_engine::STG_OUT; }
  h->cfg = *cfg;
  h->device = device;
  *out = h;   // returned even on failure so that vtts_last_error() is readable; caller destroys it
  return guarded(h, [&] {
    REQUIRE(cfg->precision >= 0 && cfg->precision <= 3, VTTS_ERR_INVALID, "unknown precision mode");
    if (cfg->precision >= 1) {
      void* fn = nullptr;
      cudaDriverEntryPointQueryResult qres;
      CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
      REQUIRE(fn != nullptr && qres == cudaDriverEntryPointSuccess, VTTS_ERR_CUDA, "cuTensorMapEncodeTiled is not available");
      h->encode_tiled = reinterpret_cast<vtts_engine::EncodeFn>(fn);
      CK(cudaFuncSetAttribute(conv_tc_persist_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      CK(cudaFuncSetAttribute(conv_tc_persist_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      CK(cudaFuncSetAttribute(conv_tc_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      CK(cudaFuncSetAttribute(conv_tc_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      CK(cudaFuncSetAttribute(conv_tc_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      CK(cudaFuncSetAttribute(conv_tc_kernel<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      for (int wi = 0; wi < 2; ++wi)
        for (int si = 0; si < 3; ++si) {
          const int S = 2 << si;
          cudaLaunchConfig_t lc;
          memset(&lc, 0, sizeof(lc));
          lc.gridDim = dim3(1, 1, S * 64); lc.blockDim = dim3(TC_THREADS);
          lc.dynamicSmemBytes = wi ? tc_smem_bytes<128>(16 * 1024) : tc_smem_bytes<64>(16 * 1024);
          cudaLaunchAttribute at[1];
          at[0].id = cudaLaunchAttributeClusterDimension;
          at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = S;
          lc.attrs = at; lc.numAttrs = 1;
          int nc = 0;
          cudaError_t e = wi ? cudaOccupancyMaxActiveClusters(&nc, conv_tc_kernel<128, false>, &lc) : cudaOccupancyMaxActiveClusters(&nc, conv_tc_kernel<64, false>, &lc);
          if (e != cudaSuccess) { nc = 0; cudaGetLastError(); }
          h->tc_cluster_cap[wi][si] = nc;
        }
      if (getenv("VTTS_VERBOSE"))
        fprintf(stderr, "[vtts] co-resident conv_tc clusters: BN64 %d/%d/%d  BN128 %d/%d/%d (S=2/4/8)\n", h->tc_cluster_cap[0][0], h->tc_cluster_cap[0][1],
                h->tc_cluster_cap[0][2], h->tc_cluster_cap[1][0], h->tc_cluster_cap[1][1], h->tc_cluster_cap[1][2]);
    }
    CK(cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, device));
    CK(cudaStreamCreateWithFlags(h->stream.out(), cudaStreamNonBlocking));
    for (auto& st : h->side) CK(cudaStreamCreateWithFlags(st.out(), cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(h->ev_fork.out(), cudaEventDisableTiming));
    for (auto& e : h->ev_join) CK(cudaEventCreateWithFlags(e.out(), cudaEventDisableTiming));
    for (auto& e : h->ev) CK(cudaEventCreate(e.out()));
    h->blob_floats = blob_floats;
    CK(h->d_blob.alloc(blob_floats));
    CK(cudaMemcpyAsync(h->d_blob.p, blob, blob_floats * sizeof(float), blob_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, h->stream));
    std::istringstream is(manifest);
    std::string name;
    unsigned long long off, n;
    while (is >> name >> off >> n) {
      REQUIRE(off + n <= blob_floats, VTTS_ERR_WEIGHTS, "manifest entry exceeds the blob");
      h->tensors[name] = Tensor{h->d_blob.p + off, (size_t)n};
    }
    h->tune = Tuning::from_env();
    if (const char* e = getenv("VTTS_MRF_BRANCH")) h->mrf_branch = atoi(e);
    if (const char* e = getenv("VTTS_MRF_HEAVY_FIRST")) h->mrf_heavy_first = atoi(e);
    if (const char* e = getenv("VTTS_PDL")) h->use_pdl = atoi(e) != 0;
    if (const char* e = getenv("VTTS_NO_POLL")) h->use_poll = atoi(e) == 0;
    if (const char* e = getenv("VTTS_NO_GRAPHS")) h->use_graphs = atoi(e) == 0;
    if (const char* e = getenv("VTTS_BUCKETS")) h->use_buckets = atoi(e) != 0;
    if (const char* e = getenv("VTTS_SPEC")) h->use_spec = atoi(e) != 0;
    if (const char* e = getenv("VTTS_SPEC_MARGIN")) h->spec_margin = (float)atof(e);      // (< 1 forces mispredictions: tests)
    if (const char* e = getenv("VTTS_CAPTURE_FIRST")) h->capture_on_first = atoi(e) != 0;   // 0: capture a bucket's graph on its second call          // 0: never enqueue phase 2 before the lengths are known    // 0: size everything by the exact lengths
    if (const char* e = getenv("VTTS_PREFETCH")) h->use_prefetch = atoi(e) != 0;
    REQUIRE(cfg->model_family >= VTTS_FAMILY_VITS2 && cfg->model_family <= VTTS_FAMILY_SOVITS, VTTS_ERR_INVALID, "unknown model family");
    if (cfg->model_family == VTTS_FAMILY_QUICKVC) h->bind_quickvc();
    else if (cfg->model_family == VTTS_FAMILY_T2S) h->bind_t2s();
    else if (cfg->model_family == VTTS_FAMILY_SOVITS) h->bind_sovits();
    else if (cfg->model_family == VTTS_FAMILY_STABLETTS) {
      h->bind_stabletts();
      h->bind_bert();
    }
    else h->bind_weights();
    h->build_prefetch_list();
    CK(cudaMemsetAsync(h->ensure(h->d_done_ctr, 4), 0, 4 * sizeof(int), h->stream));     // ticket counter of duration_kernel (self-resetting)
    CK(cudaFuncSetAttribute(dds_layer_kernel<DDS_TT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    CK(cudaFuncSetAttribute(attn_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, atc_smem_bytes(32)));
    CK(cudaFuncSetAttribute(attn_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, atc_smem_bytes(64)));
    CK(cudaFuncSetAttribute(attn_tc_kernel<96>, cudaFuncAttributeMaxDynamicSharedMemorySize, atc_smem_bytes(96)));
    CK(cudaFuncSetAttribute(attn_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, atc_smem_bytes(128)));
    CK(cudaFuncSetAttribute(attn_split_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATS_SMEM_MAX));
    CK(cudaFuncSetAttribute(attn_split_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATS_SMEM_MAX));
    CK(cudaFuncSetAttribute(attn_split_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATS_SMEM_MAX));
    CK(cudaFuncSetAttribute(attn_split_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATS_SMEM_MAX));
    CK(cudaFuncSetAttribute(attn_kernel<1, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(attn_kernel<1, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(attn_kernel<2, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(attn_kernel<2, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(attn_kernel<3, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(attn_kernel<3, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(attn_kernel<4, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(attn_kernel<4, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(conv_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, CONV_SMEM_MAX));
    CK(cudaFuncSetAttribute(conv_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, CONV_SMEM_MAX));
    CK(cudaFuncSetAttribute(conv_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, CONV_SMEM_MAX));
    CK(cudaFuncSetAttribute(mel_log_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MEL_SMEM_MAX));
    CK(cudaStreamSynchronize(h->stream));
  }, G_ATOMIC, ANY_FAMILY);
}

void vtts_destroy(vtts_handle h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->d_tl.p) {        // a timeline this handle left armed must not point at its buffer once that is freed
    unsigned long long* cur = nullptr;
    if (cudaMemcpyFromSymbol(&cur, g_timeline, sizeof(cur)) == cudaSuccess && cur == h->d_tl.p) {
      cur = nullptr;
      cudaMemcpyToSymbol(g_timeline, &cur, sizeof(cur));
    }
  }
  delete h;
}

int vtts_debug_live_bytes(uint64_t* device_bytes, uint64_t* pinned_bytes) {
  if (!device_bytes || !pinned_bytes) return VTTS_ERR_INVALID;
  *device_bytes = g_live_device_bytes;
  *pinned_bytes = g_live_pinned_bytes;
  return VTTS_OK;
}

static thread_local std::string g_free_err;      // last error of the handle-free entry points (vtts_maximum_path*), per thread
const char* vtts_last_error(vtts_handle h) { return h ? h->err.c_str() : g_free_err.c_str(); }

// Monotonic Alignment Search (mas.cuh).  No engine state is involved: the functions run on the current (or given) device.
static int mas_launch(float* d_value, const int* d_ty, const int* d_tx, int B, int Ty, int Tx, int* d_path, cudaStream_t st) {
  if (Tx > MAS_THREADS * MAS_MAXPT) { g_free_err = "vtts_maximum_path: T_x above " + std::to_string(MAS_THREADS * MAS_MAXPT); return VTTS_ERR_INVALID; }
  const size_t smem = (size_t)2 * Tx * sizeof(float);
  cudaError_t e = cudaMemsetAsync(d_path, 0, (size_t)B * Ty * Tx * sizeof(int), st);
  if (e == cudaSuccess) {
    mas_kernel<<<B, MAS_THREADS, smem, st>>>(d_value, d_path, d_ty, d_tx, Ty, Tx, nullptr, nullptr, nullptr, nullptr, nullptr);
    e = cudaGetLastError();
  }
  if (e != cudaSuccess) { g_free_err = std::string("vtts_maximum_path: ") + cudaGetErrorString(e); return VTTS_ERR_CUDA; }
  return VTTS_OK;
}

int vtts_maximum_path_dev(float* d_value, const int32_t* d_t_ys, const int32_t* d_t_xs, int B, int T_y, int T_x, int32_t* d_path, void* stream) {
  if (!d_value || !d_t_ys || !d_t_xs || !d_path || B <= 0 || T_y <= 0 || T_x <= 0) { g_free_err = "vtts_maximum_path_dev: bad argument"; return VTTS_ERR_INVALID; }
  return mas_launch(d_value, d_t_ys, d_t_xs, B, T_y, T_x, d_path, (cudaStream_t)stream);
}

int vtts_maximum_path(const float* neg_cent, const int32_t* t_ys, const int32_t* t_xs, int B, int T_y, int T_x, int32_t* path, int device) {
  if (!neg_cent || !t_ys || !t_xs || !path || B <= 0 || T_y <= 0 || T_x <= 0) { g_free_err = "vtts_maximum_path: bad argument"; return VTTS_ERR_INVALID; }
  for (int b = 0; b < B; ++b)
    if (t_ys[b] < 0 || t_ys[b] > T_y || t_xs[b] < 0 || t_xs[b] > T_x || t_xs[b] > t_ys[b]) {
      g_free_err = "vtts_maximum_path: lengths must satisfy 0 <= t_x <= t_y <= T_y, t_x <= T_x (utterance " + std::to_string(b) + ")";
      return VTTS_ERR_INVALID;
    }
  Buf<float> dv;
  Buf<int> dp, dl;
  const size_t n = (size_t)B * T_y * T_x;
  int rc = VTTS_OK;
  cudaError_t e = cudaSetDevice(device);
  if (e == cudaSuccess) e = dv.alloc(n);
  if (e == cudaSuccess) e = dp.alloc(n);
  if (e == cudaSuccess) e = dl.alloc((size_t)2 * B);
  if (e == cudaSuccess) e = cudaMemcpy(dv.p, neg_cent, n * sizeof(float), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(dl.p, t_ys, (size_t)B * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(dl.p + B, t_xs, (size_t)B * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) rc = mas_launch(dv.p, dl.p, dl.p + B, B, T_y, T_x, dp.p, 0);
  if (e == cudaSuccess && rc == VTTS_OK) e = cudaMemcpy(path, dp.p, n * sizeof(int), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) { g_free_err = std::string("vtts_maximum_path: ") + cudaGetErrorString(e); return VTTS_ERR_CUDA; }
  return rc;
}

int vtts_durations(vtts_handle h, const int64_t* ids, const int64_t* lengths, const int64_t* sid, int B, int t_max,
                   const float* scales, const float* noise_dp, uint64_t seed, int64_t* y_lengths, int32_t* durations) {
  if (!ids || !lengths || !sid || !scales || !y_lengths) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_durations(h, ids, lengths, sid, B, t_max, scales, noise_dp, seed, y_lengths, durations); }, G_BEGIN);
}

int vtts_synthesize(vtts_handle h, const float* noise_z, int z_ld, float* wav, int64_t wav_ld, int32_t* frame_token, int idx_ld) {
  if (!wav) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_synthesize(h, noise_z, z_ld, wav, wav_ld, frame_token, idx_ld); }, G_CONT);
}

int vtts_durations_dev(vtts_handle h, const int64_t* d_ids, const int64_t* lengths_host, const int64_t* d_sid, int B, int t_max,
                       const float* scales, const float* d_noise_dp, uint64_t seed, int64_t* y_lengths_host) {
  if (!d_ids || !lengths_host || !d_sid || !scales || !y_lengths_host) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_durations_dev(h, d_ids, lengths_host, d_sid, B, t_max, scales, d_noise_dp, seed, y_lengths_host); }, G_BEGIN);
}

int vtts_synthesize_dev(vtts_handle h, const float* d_noise_z, int z_ld, float* d_wav, int64_t wav_ld) {
  if (!d_wav) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_synthesize_dev(h, d_noise_z, z_ld, d_wav, wav_ld); }, G_CONT);
}

// ---- streaming: flow once, then decode halo-extended chunks (SURVEY.md section 5: the decoder's receptive field is
// +-23.9 latent frames, so a chunk decoded with a 24-frame halo on each side reproduces the monolithic output).
int vtts_decoder_halo(vtts_handle h) { return h ? 24 : 0; }

int vtts_flow(vtts_handle h, const float* noise_z, int z_ld) {
  return guarded(h, [&] {
    REQUIRE(h->have_durations, VTTS_ERR_STATE, "vtts_flow called without vtts_durations");
    REQUIRE(!noise_z || z_ld >= h->real_maxFrm, VTTS_ERR_CAPACITY, "noise_z has fewer columns than max(y_lengths)");
    if (noise_z) h->stage_noise_z(noise_z, z_ld);
    h->last_graphed = false;
    h->phase2(noise_z, z_ld, false, /*run_decoder=*/false);
    CK(cudaStreamSynchronize(h->stream));
    h->have_durations = false;
    h->have_latent = true;
  }, G_CONT);
}

int vtts_decode_chunk(vtts_handle h, int f0, int f1, float* wav, int64_t wav_capacity) {
  if (!wav) return VTTS_ERR_INVALID;
  return guarded(h, [&] {
    REQUIRE(h->have_latent, VTTS_ERR_STATE, "vtts_decode_chunk called without vtts_flow");
    REQUIRE(h->B == 1, VTTS_ERR_INVALID, "chunked decoding handles one utterance per call");
    const int T = h->h_frm_len[0];
    REQUIRE(0 <= f0 && f0 < f1 && f1 <= T, VTTS_ERR_INVALID, "chunk out of range");
    REQUIRE((int64_t)(f1 - f0) * h->hop <= wav_capacity, VTTS_ERR_CAPACITY, "chunk does not fit the output buffer");
    const int halo = 24;
    const int lo = std::max(0, f0 - halo), hi = std::min(T, f1 + halo);
    int* dc = h->ensure(h->d_chunk, 4);
    vtts_engine::Staging& st = h->stg[vtts_engine::STG_CHUNK];
    st.begin();
    st.add(h->d_chunk, 3);
    st.commit();
    int* pin = st.host(h->d_chunk);
    pin[0] = hi - lo; pin[1] = lo; pin[2] = hi;
    st.upload();
    // the launches size grids and split-K for the chunk (the planes keep the full utterance's row count, Tfrm: the chunk is
    // addressed by its absolute rows)
    const Rows r{dc, dc + 1, 1, hi - lo, {hi - lo}, {hi - lo}, h->tune};
    h->last_graphed = false;
    h->decode(h->d_z.p, r);
    const size_t n = (size_t)(f1 - f0) * h->hop;
    memcpy(wav, read_back(h, h->d_wav, n, 0, (size_t)f0 * h->hop), n * sizeof(float));
  });
}

int vtts_infer(vtts_handle h, const int64_t* ids, const int64_t* lengths, const int64_t* sid, int B, int t_max, const float* scales,
               const float* noise_dp, const float* noise_z, int z_ld, uint64_t seed, int64_t* y_lengths, float* wav, int64_t wav_ld,
               int32_t* frame_token, int idx_ld) {
  if (!ids || !lengths || !sid || !scales || !y_lengths || !wav) return VTTS_ERR_INVALID;
  int phase = 0;
  const int rc = guarded(h, [&] {
    impl_infer(h, ids, lengths, sid, B, t_max, scales, noise_dp, noise_z, z_ld, seed, y_lengths, wav, wav_ld, frame_token, idx_ld, &phase);
  });
  if (rc == VTTS_ERR_CAPACITY && phase == 1) {      // durations are kept: this thread may finish with vtts_synthesize
    std::lock_guard<std::mutex> lk(h->mu);
    h->two_phase = true;
    h->owner = std::this_thread::get_id();
  }
  return rc;
}

int vtts_infer_dev(vtts_handle h, const int64_t* d_ids, const int64_t* lengths_host, const int64_t* d_sid, int B, int t_max,
                   const float* scales, const float* d_noise_dp, const float* d_noise_z, int z_ld, uint64_t seed,
                   int64_t* y_lengths_host, float* d_wav, int64_t wav_ld) {
  if (!d_ids || !lengths_host || !d_sid || !scales || !y_lengths_host || !d_wav) return VTTS_ERR_INVALID;
  int phase = 0;
  const int rc = guarded(h, [&] {
    impl_infer_dev(h, d_ids, lengths_host, d_sid, B, t_max, scales, d_noise_dp, d_noise_z, z_ld, seed, y_lengths_host, d_wav, wav_ld, &phase);
  });
  if (rc == VTTS_ERR_CAPACITY && phase == 1) {
    std::lock_guard<std::mutex> lk(h->mu);
    h->two_phase = true;
    h->owner = std::this_thread::get_id();
  }
  return rc;
}

int vtts_convert(vtts_handle h, const float* wav, const int64_t* wav_lengths, int B, int64_t wav_ld, const int64_t* sid_src,
                 const int64_t* sid_tgt, float noise_scale, const float* noise_q, int q_ld, uint64_t seed, float* out_wav,
                 int64_t out_ld, int64_t* out_frames) {
  if (!wav || !wav_lengths || !sid_src || !sid_tgt || !out_wav || !out_frames) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_convert(h, false, wav, wav_lengths, B, wav_ld, sid_src, sid_tgt, noise_scale, noise_q, q_ld, seed, out_wav,
                                       out_ld, out_frames); });
}

int vtts_convert_spec(vtts_handle h, const float* spec, const int64_t* spec_lengths, int B, int64_t spec_ld, const int64_t* sid_src,
                      const int64_t* sid_tgt, float noise_scale, const float* noise_q, int q_ld, uint64_t seed, float* out_wav,
                      int64_t out_ld, int64_t* out_frames) {
  if (!spec || !spec_lengths || !sid_src || !sid_tgt || !out_wav || !out_frames) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_convert(h, true, spec, spec_lengths, B, spec_ld, sid_src, sid_tgt, noise_scale, noise_q, q_ld, seed,
                                       out_wav, out_ld, out_frames); });
}

int vtts_align(vtts_handle h, const int64_t* ids, const int64_t* id_lengths, int t_max, const int64_t* sid, const float* wav,
               const int64_t* wav_lengths, int B, int64_t wav_ld, float noise_scale, const float* noise_q, int q_ld, uint64_t seed,
               int32_t* durations, int32_t* token_of_frame, int64_t tof_ld, float* score, int64_t* out_frames) {
  if (!ids || !id_lengths || !wav || !wav_lengths || !durations || !out_frames) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_align(h, false, ids, id_lengths, t_max, sid, wav, wav_lengths, B, wav_ld, noise_scale, noise_q, q_ld, seed,
                                     durations, token_of_frame, tof_ld, score, out_frames); });
}

int vtts_align_spec(vtts_handle h, const int64_t* ids, const int64_t* id_lengths, int t_max, const int64_t* sid, const float* spec,
                    const int64_t* spec_lengths, int B, int64_t spec_ld, float noise_scale, const float* noise_q, int q_ld, uint64_t seed,
                    int32_t* durations, int32_t* token_of_frame, int64_t tof_ld, float* score, int64_t* out_frames) {
  if (!ids || !id_lengths || !spec || !spec_lengths || !durations || !out_frames) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_align(h, true, ids, id_lengths, t_max, sid, spec, spec_lengths, B, spec_ld, noise_scale, noise_q, q_ld,
                                     seed, durations, token_of_frame, tof_ld, score, out_frames); });
}

int vtts_hop(vtts_handle h) { return h ? h->hop : 0; }

int vtts_stage_timings(vtts_handle h, float* ms, int n) {
  if (!h || !ms) return VTTS_ERR_INVALID;
  for (int i = 0; i < n && i < 8; ++i) ms[i] = h->stage_ms[i];
  return VTTS_OK;
}

uint64_t vtts_kernel_launches(vtts_handle h) { return h ? h->launches : 0; }
void* vtts_stream(vtts_handle h) { return h ? (void*)h->stream : nullptr; }

int vtts_set_graphs(vtts_handle h, int enable) {
  return guarded(h, [&] { h->use_graphs = enable != 0; }, G_ATOMIC, ANY_FAMILY);
}

uint64_t vtts_graph_replays(vtts_handle h) { return h ? h->graph_replays : 0; }

int vtts_host_timings(vtts_handle h, double* us, int n) {
  if (!h || !us) return VTTS_ERR_INVALID;
  for (int i = 0; i < n && i < 8; ++i) us[i] = h->host_us[i];
  return VTTS_OK;
}

int vtts_speculation_stats(vtts_handle h, uint64_t* hits, uint64_t* misses) {
  if (!h || !hits || !misses) return VTTS_ERR_INVALID;
  *hits = h->spec_hits;
  *misses = h->spec_misses;
  return VTTS_OK;
}

int vtts_profile(vtts_handle h, int enable) {
  return guarded(h, [&] {
    h->profiling = enable != 0;
    h->prof_used = 0;
    h->prof_flops = 0.0;
    h->prof_launches = 0;
    h->tc_prof_used = 0;
    h->tc_prof_flops = 0.0;
    h->tc_prof_launches = 0;
  }, G_ATOMIC, ANY_FAMILY);
}

int vtts_profile_read(vtts_handle h, double* conv_ms, uint64_t* conv_launches, double* conv_flops) {
  if (!conv_ms || !conv_launches || !conv_flops) return VTTS_ERR_INVALID;
  return guarded(h, [&] {
    CK(cudaStreamSynchronize(h->stream));
    double ms = 0.0;
    for (size_t i = 0; i + 1 < h->prof_used; i += 2) {
      float t = 0.f;
      CK(cudaEventElapsedTime(&t, h->prof_ev[i], h->prof_ev[i + 1]));
      ms += t;
    }
    *conv_ms = ms;
    *conv_launches = h->prof_launches;
    *conv_flops = h->prof_flops;
  }, G_ATOMIC, ANY_FAMILY);
}

// Timeline: enable -> every kernel's first CTA appends (source line, globaltimer) to a device buffer; read returns pairs.
int vtts_timeline(vtts_handle h, int enable, unsigned long long* out, size_t max_pairs, size_t* n_out) {
  return guarded(h, [&] {
    CK(cudaStreamSynchronize(h->stream));
    if (enable == 1) {
      if (!h->d_tl.p) CK(h->d_tl.alloc(1 + 2 * 4000));
      CK(cudaMemset(h->d_tl.p, 0, (1 + 2 * 4000) * 8));
      CK(cudaMemcpyToSymbol(g_timeline, &h->d_tl.p, sizeof(h->d_tl.p)));
    } else if (enable == 0) {
      unsigned long long* z = nullptr;
      CK(cudaMemcpyToSymbol(g_timeline, &z, sizeof(z)));
    } else if (h->d_tl.p && out && n_out) {
      std::vector<unsigned long long> hbuf(1 + 2 * 4000);
      CK(cudaMemcpy(hbuf.data(), h->d_tl.p, hbuf.size() * 8, cudaMemcpyDeviceToHost));
      size_t n = std::min<size_t>((size_t)hbuf[0], std::min<size_t>(4000, max_pairs));
      memcpy(out, hbuf.data() + 1, n * 16);
      *n_out = n;
    }
  }, G_ATOMIC, ANY_FAMILY);
}

int vtts_debug_flags(vtts_handle h, int flags) {
  if (!h) return VTTS_ERR_INVALID;
  h->debug_flags = flags;
  return VTTS_OK;
}

int vtts_debug_read(vtts_handle h, const char* name, float* out, size_t max_floats, size_t* n_out) {
  if (!name || !out || !n_out) return VTTS_ERR_INVALID;
  return guarded(h, [&] {
    const vtts_config& c = h->cfg;
    const std::string nm(name);
    const float* src = nullptr;
    size_t n = 0;
    const size_t T = h->real_Ttok, F = h->real_Tfrm;
    if (nm == "x") { src = h->d_x.p; n = T * c.hidden_channels; }
    else if (nm == "stats") { src = h->d_stats.p; n = T * 2 * c.inter_channels; }
    else if (nm == "dx") { src = h->d_dx.p; n = T * c.dp_filter_channels; }
    else if (nm == "za") { src = h->d_za.p; n = T; }
    else if (nm == "zb") { src = h->d_zb.p; n = T; }
    else if (nm == "condv") { src = h->d_condv.p; n = (size_t)h->B * h->condR; }
    else if (nm == "z_p") { src = h->d_zp_dbg.p; n = F * c.inter_channels; }
    else if (nm == "z") { src = h->d_z.p; n = F * c.inter_channels; }
    else if (nm == "d0") { src = h->d_d0.p; n = F * c.upsample_initial_channel; }
    else if (nm == "vc_spec") { src = h->d_vfeat.p; n = F * h->spec_pad; }
    else if (nm == "vc_z") { src = h->d_vz_dbg.p; n = F * c.inter_channels; }
    else if (nm == "vc_z_p") { src = h->d_vzp_dbg.p; n = F * c.inter_channels; }
    else if (nm == "vc_z_hat") { src = h->d_z.p; n = F * c.inter_channels; }
    else if (nm == "align_neg_cent") { src = h->d_ncent_dbg.p; n = (size_t)h->B * h->real_maxFrm * h->real_maxTok; }
    else if (nm == "post") { src = h->d_post.p; n = (F * h->up_total + h->B) * c.subbands * (c.istft_n_fft + 2); }
    else if (nm == "spk_x0") { src = h->d_sx[0].p; n = F * SPK_GATES; }
    else if (nm == "spk_x1" || nm == "spk_x2") { src = h->d_sx[nm[5] - '0'].p; n = (size_t)h->spk_rows * SPK_GATES; }
    else if (nm == "spk_h0" || nm == "spk_h1" || nm == "spk_h2") { src = h->d_sh[nm[5] - '0'].p; n = (size_t)h->spk_rows * SPK_H; }
    else if (nm == "spk_g") { src = h->d_sg.p; n = (size_t)h->B * SPK_H; }
    else if (nm == "cv_feat") { src = h->d_cvl[(c.cv_n_conv - 1) & 1].p; n = (size_t)h->cvp.tot0 / h->cv_P * c.cv_conv_dim; }
    else if (nm == "cv_gn_sum") { src = h->d_cvps.p; n = (size_t)h->B * h->cvp.MC * c.cv_conv_dim; }
    else if (nm == "cv_gn_sq") { src = h->d_cvpq.p; n = (size_t)h->B * h->cvp.MC * c.cv_conv_dim; }
    else if (nm == "st_film") { src = h->d_stfilm.p; n = (size_t)h->stp.steps * c.st_layers * 2 * c.st_hidden; }
    else if (nm == "st_ada") { src = h->d_stada.p; n = (size_t)h->stp.NS * c.st_layers * 6 * c.st_hidden; }
    else if (nm == "st_cond") { src = h->d_stxc.p; n = (size_t)h->stp.Ttot * (c.st_noise + c.st_hidden); }
    else if (nm == "st_rope") { src = h->d_strope.p; n = (size_t)h->maxFrm * (c.st_hidden / c.st_heads / 2); }
    else if (nm == "st_norm1") { src = h->d_stdbg_n.p; n = (size_t)h->stp.Ttot * c.st_hidden; }
    else if (nm == "st_qkv") { src = h->d_stdbg_qkv.p; n = (size_t)h->stp.Ttot * 3 * c.st_hidden; }
    else if (nm == "st_mu") { src = h->d_stmu.p; n = (size_t)h->stp.Ttot * c.st_cond; }
    else if (nm == "st_tok_x") { src = h->d_sttx.p; n = T * c.st_cond; }
    else if (nm == "st_mu_dp") { src = h->d_stmudp.p; n = T * c.st_dur_channels; }
    else if (nm == "st_logw") { src = h->d_stlogw.p; n = T; }
    else if (nm == "cv_enc_in") { src = h->d_cvdbg.p; n = (size_t)h->cvp.tot0 / h->cv_P * c.cv_hidden; }
    else if (nm == "sv_proj") { src = h->d_svproj.p; n = (size_t)h->svp.pairs_cap * c.cv_hidden; }
    else if (nm.rfind("stage", 0) == 0) {
      const int i = atoi(nm.c_str() + 5);
      REQUIRE(i >= 0 && i < (int)h->d_stage.size(), VTTS_ERR_INVALID, "no such stage");
      int rm = 1, ch = c.upsample_initial_channel;
      for (int j = 0; j <= i; ++j) { rm *= c.upsample_rates[j]; ch /= 2; }
      src = h->d_stage[i].p; n = F * rm * ch;
    }
    else if (h->st_taps.count(nm)) { src = h->st_taps[nm].buf.p; n = h->st_taps[nm].n; }
    REQUIRE(src != nullptr, VTTS_ERR_INVALID, "unknown or unallocated debug tensor");
    REQUIRE(n <= max_floats, VTTS_ERR_CAPACITY, "debug buffer too small");
    CK(cudaMemcpyAsync(out, src, n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    *n_out = n;
  }, G_ATOMIC, ANY_FAMILY);
}

int vtts_sovits_semantic(vtts_handle h, const float* wav, const int64_t* wav_lengths, int B, int64_t wav_ld, int64_t* codes,
                         int64_t codes_ld, int64_t* out_frames) {
  if (!wav || !wav_lengths || !codes || !out_frames) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_sovits(h, wav, nullptr, wav_lengths, B, wav_ld, codes, codes_ld, out_frames); }, G_ATOMIC,
                 VTTS_FAMILY_SOVITS);
}

int vtts_sovits_latent(vtts_handle h, const float* feats, const int64_t* frames, int B, int64_t feats_ld, int64_t* codes,
                       int64_t codes_ld, int64_t* out_frames) {
  if (!feats || !frames || !codes || !out_frames) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_sovits(h, nullptr, feats, frames, B, feats_ld, codes, codes_ld, out_frames); }, G_ATOMIC,
                 VTTS_FAMILY_SOVITS);
}

int vtts_speaker_embedding(vtts_handle h, const float* wav, const int64_t* wav_lengths, int B, int64_t wav_ld, float* g_out) {
  if (!wav || !wav_lengths || !g_out) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_speaker_embedding(h, false, wav, wav_lengths, B, wav_ld, g_out); }, G_ATOMIC, VTTS_FAMILY_QUICKVC);
}

int vtts_speaker_embedding_mel(vtts_handle h, const float* mel, const int64_t* mel_lengths, int B, int64_t mel_ld, float* g_out) {
  if (!mel || !mel_lengths || !g_out) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_speaker_embedding(h, true, mel, mel_lengths, B, mel_ld, g_out); }, G_ATOMIC, VTTS_FAMILY_QUICKVC);
}

int vtts_quickvc_convert(vtts_handle h, const float* units, const int64_t* unit_lengths, int B, int64_t units_ld, const float* g,
                         float noise_scale, const float* noise, int noise_ld, uint64_t seed, float* out_wav, int64_t out_ld,
                         int64_t* out_frames) {
  if (!units || !unit_lengths || !out_wav || !out_frames) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_quickvc_convert(h, units, nullptr, unit_lengths, B, units_ld, g, noise_scale, noise, noise_ld, seed, out_wav,
                                               out_ld, out_frames); }, G_ATOMIC, VTTS_FAMILY_QUICKVC);
}

int vtts_content_units(vtts_handle h, const float* wav, const int64_t* wav_lengths, int B, int64_t wav_ld, float* units,
                       int64_t units_ld, int64_t* out_frames) {
  if (!wav || !wav_lengths || !units || !out_frames) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_content_units(h, wav, wav_lengths, B, wav_ld, units, units_ld, out_frames); }, G_ATOMIC, VTTS_FAMILY_QUICKVC);
}

int vtts_bert_features(vtts_handle h, const int64_t* ids, const int64_t* lengths, int B, int64_t ids_ld, float* out, int64_t out_ld) {
  if (!ids || !lengths || !out) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_bert_features(h, ids, lengths, B, ids_ld, out, out_ld); }, G_ATOMIC, VTTS_FAMILY_STABLETTS);
}

int vtts_t2s_decode(vtts_handle h, const int64_t* ids, const int64_t* lengths, int B, int64_t ids_ld, const float* bert,
                    const int64_t* prompts, const int64_t* prompt_lengths, int64_t prompts_ld, int top_k, float top_p, float temperature,
                    float repetition_penalty, int early_stop_num, int step_cap, const uint64_t* seeds, const float* q, int64_t q_ld,
                    int64_t* tokens, int64_t tokens_ld, int64_t* n_tokens, int64_t* idx, float* logits, int64_t logits_ld) {
  return guarded(h, [&] { impl_t2s_decode(h, ids, lengths, B, ids_ld, bert, prompts, prompt_lengths, prompts_ld, top_k, top_p, temperature,
                                          repetition_penalty, early_stop_num, step_cap, seeds, q, q_ld, tokens, tokens_ld, n_tokens, idx,
                                          logits, logits_ld); }, G_ATOMIC, VTTS_FAMILY_T2S);
}

int vtts_quickvc_convert_wav(vtts_handle h, const float* wav, const int64_t* wav_lengths, int B, int64_t wav_ld, const float* g,
                             float noise_scale, const float* noise, int noise_ld, uint64_t seed, float* out_wav, int64_t out_ld,
                             int64_t* out_frames) {
  if (!wav || !wav_lengths || !out_wav || !out_frames) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_quickvc_convert(h, nullptr, wav, wav_lengths, B, wav_ld, g, noise_scale, noise, noise_ld, seed, out_wav,
                                               out_ld, out_frames); }, G_ATOMIC, VTTS_FAMILY_QUICKVC);
}

int vtts_cfm_decode(vtts_handle h, const float* mu, const int64_t* lengths, int B, int64_t mu_ld, const int64_t* sid,
                    const float* spk_rows, int n_timesteps, float temperature, float guidance_scale, const float* noise,
                    int64_t noise_ld, uint64_t seed, float* mel_out, int64_t mel_ld, int denormalise) {
  if (!mu || !lengths || !mel_out) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_cfm_decode(h, mu, lengths, B, mu_ld, sid, spk_rows, n_timesteps, temperature, guidance_scale, noise, noise_ld,
                                          seed, mel_out, mel_ld, denormalise); }, G_ATOMIC, VTTS_FAMILY_STABLETTS);
}

int vtts_stabletts_synthesise(vtts_handle h, const int64_t* ids, const int64_t* id_lengths, int B, int64_t t_max, const float* bert,
                              const float* pause, const int64_t* sid, int n_timesteps, float temperature, float length_scale,
                              float guidance_scale, const float* noise, int64_t noise_ld, uint64_t seed, float* mel_out, int64_t mel_ld,
                              int64_t* mel_lengths, int32_t* durations, float* prior_out, int denormalise) {
  if (!ids || !id_lengths || !bert || !sid || !mel_out || !mel_lengths) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_stabletts_synthesise(h, ids, id_lengths, B, t_max, bert, pause, sid, n_timesteps, temperature, length_scale,
                                                    guidance_scale, noise, noise_ld, seed, mel_out, mel_ld, mel_lengths, durations, prior_out,
                                                    denormalise); }, G_ATOMIC, VTTS_FAMILY_STABLETTS);
}

int vtts_stabletts_synthesise_wav(vtts_handle h, const int64_t* ids, const int64_t* id_lengths, int B, int64_t t_max, const float* bert,
                                  const float* pause, const int64_t* sid, int n_timesteps, float temperature, float length_scale,
                                  float guidance_scale, const float* noise, int64_t noise_ld, uint64_t seed, float* mel_out, int64_t mel_ld,
                                  int64_t* mel_lengths, int32_t* durations, float* prior_out, int denormalise, float* wav, int64_t wav_ld,
                                  int64_t* wav_lengths) {
  if (!ids || !id_lengths || !bert || !sid || !mel_lengths || !wav || !wav_lengths || (prior_out && !mel_out)) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_stabletts_synthesise(h, ids, id_lengths, B, t_max, bert, pause, sid, n_timesteps, temperature, length_scale,
                                                    guidance_scale, noise, noise_ld, seed, mel_out, mel_ld, mel_lengths, durations, prior_out,
                                                    denormalise, wav, wav_ld, wav_lengths); }, G_ATOMIC, VTTS_FAMILY_STABLETTS);
}

int vtts_stabletts_synthesise_pieces_wav(vtts_handle h, const int64_t* ids, const int64_t* id_lengths, int B, int64_t t_max,
                                         const int64_t* pieces, const int64_t* piece_lengths, int64_t pieces_ld, const int32_t* bert_rows,
                                         const float* pause, const int64_t* sid, int n_timesteps, float temperature, float length_scale,
                                         float guidance_scale, const float* noise, int64_t noise_ld, uint64_t seed, float* mel_out,
                                         int64_t mel_ld, int64_t* mel_lengths, int32_t* durations, float* prior_out, int denormalise, float* wav,
                                         int64_t wav_ld, int64_t* wav_lengths) {
  if (!ids || !id_lengths || !pieces || !piece_lengths || !bert_rows || !sid || !mel_lengths || !wav || !wav_lengths || (prior_out && !mel_out))
    return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_stabletts_synthesise(h, ids, id_lengths, B, t_max, nullptr, pause, sid, n_timesteps, temperature, length_scale,
                                                    guidance_scale, noise, noise_ld, seed, mel_out, mel_ld, mel_lengths, durations, prior_out,
                                                    denormalise, wav, wav_ld, wav_lengths, pieces, piece_lengths, pieces_ld, bert_rows); },
                 G_ATOMIC, VTTS_FAMILY_STABLETTS);
}

int vtts_hifigan_vocode(vtts_handle h, const float* mel, const int64_t* mel_lengths, int B, int64_t mel_ld, float* wav, int64_t wav_ld,
                        int64_t* wav_lengths) {
  if (!mel || !mel_lengths || !wav || !wav_lengths) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_hifigan_vocode(h, mel, mel_lengths, B, mel_ld, wav, wav_ld, wav_lengths); }, G_ATOMIC, VTTS_FAMILY_STABLETTS);
}

int vtts_resample(vtts_handle h, const float* wav, const int64_t* lengths, int B, int64_t ld, int from_rate, int to_rate,
                  float trim_top_db, float* out, int64_t out_ld, int64_t* out_lengths, int64_t* trim_bounds) {
  return guarded(h, [&] { impl_resample(h, wav, lengths, B, ld, from_rate, to_rate, trim_top_db, out, out_ld, out_lengths, trim_bounds); },
                 G_ATOMIC, ANY_FAMILY);
}

// A device copy of a debug hook's host argument, held by `dev` (so freed on every exit).
static void* upload(std::vector<Buf<char>>& dev, const void* src, size_t bytes, cudaStream_t s) {
  Buf<char>& d = dev.emplace_back();
  CK(d.alloc(std::max<size_t>(bytes, 16)));
  if (src) CK(cudaMemcpyAsync(d.p, src, bytes, cudaMemcpyHostToDevice, s));
  return d.p;
}

// Unit-test hook of the attention kernels (include/vtts.h): one launch through launch_attn_tc / launch_attn on host tensors.
int vtts_debug_attention(vtts_handle h, const char* layer, int B, const int* lens, const int* launch_lens, const float* qkv,
                         size_t rows, int kernel, float* out, uint16_t* planes, int p_planes, int iters, float* ms_out,
                         vtts_attn_report* report) {
  return guarded(h, [&] {
    REQUIRE(layer && lens && qkv && B >= 1, VTTS_ERR_INVALID, "debug_attention: missing layer, lengths or input");
    REQUIRE(out || planes, VTTS_ERR_INVALID, "debug_attention: neither fp32 output nor output planes requested");
    REQUIRE(!planes || p_planes == 2 || p_planes == 3, VTTS_ERR_INVALID, "debug_attention: the output has 2 or 3 planes");
    REQUIRE(kernel >= VTTS_ATTN_AUTO && kernel <= VTTS_ATTN_FFMA, VTTS_ERR_INVALID, "debug_attention: unknown kernel selection");
    const std::string nm(layer);
    const EncLayerW* L = nullptr;
    if (nm.rfind("enc.", 0) == 0) {
      const int i = atoi(nm.c_str() + 4);
      REQUIRE(i >= 0 && i < (int)h->enc.size(), VTTS_ERR_INVALID, "no such encoder layer");
      L = &h->enc[i];
    } else if (nm.rfind("flow.", 0) == 0) {
      const int f = atoi(nm.c_str() + 5);
      REQUIRE(f >= 0 && f < (int)h->flow.size() && h->cfg.use_transformer_flows, VTTS_ERR_INVALID, "no such flow layer");
      L = &h->flow[f].tr;
    }
    REQUIRE(L != nullptr, VTTS_ERR_INVALID, "layer must be enc.<i> or flow.<f>.tr");
    const int H = h->cfg.hidden_channels;
    std::vector<int> ll(B);
    std::vector<long> off(B + 1, 0);
    int maxLen = 0;
    for (int b = 0; b < B; ++b) {
      REQUIRE(lens[b] >= 1, VTTS_ERR_INVALID, "debug_attention: lengths must be >= 1");
      ll[b] = launch_lens ? launch_lens[b] : lens[b];
      REQUIRE(ll[b] >= lens[b], VTTS_ERR_INVALID, "debug_attention: launch lengths must be >= the lengths");
      off[b + 1] = off[b] + lens[b] + (b + 1 < B ? SEQ_GAP : 0);
      maxLen = std::max(maxLen, ll[b]);
    }
    REQUIRE((long)rows >= off[B], VTTS_ERR_INVALID, "debug_attention: qkv has fewer rows than the packed utterances");
    // planes() and flush_tails() read the member B: restored on every exit
    struct KeepB { vtts_engine* h; int B; ~KeepB() { h->B = B; } } keep{h, h->B};
    h->B = B;
    // the heuristics see the launch lengths; the device lengths are set below
    Rows r{nullptr, nullptr, B, maxLen, ll, std::vector<int>(lens, lens + B), h->tune.with_attention(kernel)};
    // ---- kernel selection (refused before anything is launched)
    bool use_tc = false;
    switch (kernel) {
      case VTTS_ATTN_AUTO: use_tc = h->attn_use_tc(*L, H, r); break;
      case VTTS_ATTN_TC:
        REQUIRE(h->attn_tc_ok(*L, H, r.tune), VTTS_ERR_INVALID, "debug_attention: tensor-core attention is not available for this layer (relative tables / window)");
        use_tc = true;
        break;
      case VTTS_ATTN_SPLIT:
        REQUIRE(h->attn_split_fits(*L, H, r), VTTS_ERR_INVALID, "debug_attention: the split-KV kernel does not fit this launch");
        break;
      default: break;                               // R1 / R4 / FFMA: launch_attn's choice under that tuning
    }
    REQUIRE(!(use_tc && planes && p_planes != 2), VTTS_ERR_INVALID, "debug_attention: the tensor-core kernel writes 2 output planes");
    // ---- device copies
    std::vector<Buf<char>> dev;
    cudaStream_t st = h->stream;
    CK(cudaStreamSynchronize(st));
    std::vector<int> lo(2 * B + 3);
    for (int b = 0; b < B; ++b) lo[b] = lens[b];
    for (int b = 0; b <= B; ++b) lo[B + b] = (int)off[b];
    lo[2 * B + 1] = (int)rows; lo[2 * B + 2] = 0;   // all rows as one span (input split)
    int* dl = static_cast<int*>(upload(dev, lo.data(), lo.size() * sizeof(int), st));
    const int* dlens = dl;
    const int* doffs = dl + B;
    r.lens = dlens; r.offs = doffs;
    const float* dq = static_cast<const float*>(upload(dev, qkv, rows * 3 * H * sizeof(float), st));
    float* dout = static_cast<float*>(upload(dev, out, rows * H * sizeof(float), st));   // (the FFMA kernels always write fp32)
    const size_t pn = rows * H;
    Planes po;
    if (planes) {
      __nv_bfloat16* dp = static_cast<__nv_bfloat16*>(upload(dev, planes, (size_t)p_planes * pn * 2, st));
      po.hi = dp; po.mid = p_planes == 3 ? dp + pn : nullptr; po.lo = dp + (p_planes - 1) * pn; po.C = H; po.rows = (long)rows;
    }
    Planes pq;
    if (use_tc) {
      // split every row on the device, then the production zero_tails pass: gap rows and rows behind each utterance hold the
      // caller's data until that pass clears them, as in a phase
      h->begin_planes();
      pq = h->planes(58, (long)rows, 1, 3 * H);
      h->klaunch(split_planes_kernel, dim3((unsigned)((rows + EW_ROWS - 1) / EW_ROWS), 1), dim3(EW_THREADS), (size_t)0, dq, 3 * H, pq.hi,
                 pq.lo, 3 * H, 3 * H, 1.f, 0, 1, (const int*)(dl + 2 * B + 1), (const int*)(dl + 2 * B + 2));
      h->flush_tails(dlens, doffs);
    }
    auto once = [&] {
      if (use_tc) h->launch_attn_tc(pq, out ? dout : nullptr, planes ? &po : nullptr, *L, H, r);
      else h->launch_attn(dq, dout, *L, H, planes ? &po : nullptr, r);
    };
    once();
    CK(cudaStreamSynchronize(st));
    if (out) CK(cudaMemcpy(out, dout, rows * H * sizeof(float), cudaMemcpyDeviceToHost));
    if (planes) CK(cudaMemcpy(planes, po.hi, (size_t)p_planes * pn * 2, cudaMemcpyDeviceToHost));
    if (report) *report = h->last_attn;
    if (iters > 0 && ms_out) {
      Event e0, e1;
      CK(cudaEventCreate(e0.out())); CK(cudaEventCreate(e1.out()));
      CK(cudaEventRecord(e0, st));
      for (int i = 0; i < iters; ++i) once();
      CK(cudaEventRecord(e1, st));
      CK(cudaStreamSynchronize(st));
      float ms = 0.f;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      *ms_out = ms / iters;
    }
  });
}

// Unit-test hook of the dense conv kernels (include/vtts.h): one grouped launch through launch_tc / launch_conv on host tensors.
int vtts_debug_conv(vtts_handle h, int use_tc, int B, const int* lens, int rmul, int n_problems, const vtts_conv_problem* problems,
                    const void* x, size_t x_n, int x_planes, float* y, size_t y_n, const float* res, size_t res_n, uint16_t* p_out,
                    size_t p_n, int p_planes, const vtts_conv_overrides* ov, vtts_conv_report* report) {
  return guarded(h, [&] {
    REQUIRE(lens && problems && x && B >= 1 && rmul >= 1, VTTS_ERR_INVALID, "debug_conv: missing lengths, problems or input");
    REQUIRE(n_problems >= 1 && n_problems <= TC_MAXP && n_problems <= CV_MAXP, VTTS_ERR_INVALID, "debug_conv: 1..4 problems per launch");
    REQUIRE(!use_tc || h->encode_tiled, VTTS_ERR_INVALID, "debug_conv: the tensor-core conv needs a precision >= 1 engine");
    std::vector<long> off(B + 1, 0);
    int maxLen = 0;
    for (int b = 0; b < B; ++b) {
      REQUIRE(lens[b] >= 1, VTTS_ERR_INVALID, "debug_conv: lengths must be >= 1");
      off[b + 1] = off[b] + lens[b] + (b + 1 < B ? SEQ_GAP : 0);
      maxLen = std::max(maxLen, lens[b]);
    }
    const long gap = (long)SEQ_GAP * rmul;
    const vtts_conv_problem& P0 = problems[0];
    if (use_tc) {
      REQUIRE(x_planes == 2 || x_planes == 3, VTTS_ERR_INVALID, "debug_conv: the tensor-core input has 2 or 3 planes");
    }
    bool any_planes = false;
    for (int i = 0; i < n_problems; ++i) {
      const vtts_conv_problem& q = problems[i];
      REQUIRE(q.Cin > 0 && q.Cout > 0 && q.k >= 1 && q.dil >= 1 && q.pad >= 0 && q.out_mul >= 1 && q.out_add >= 0 && q.in_extra >= 0 &&
                  q.out_seq_extra >= 0 && q.bias,
              VTTS_ERR_INVALID, "debug_conv: bad problem geometry or missing bias");
      REQUIRE((q.epi & ~(use_tc ? (TCE_RELU | TCE_GATE) : (EPI_RELU | EPI_GATE | EPI_TANH))) == 0, VTTS_ERR_INVALID, "debug_conv: unknown epilogue");
      REQUIRE(!(q.epi & EPI_GATE) || q.Cout % 2 == 0, VTTS_ERR_INVALID, "debug_conv: the gate needs an even Cout");
      REQUIRE(!q.cond || q.cond_ld >= q.Cout, VTTS_ERR_INVALID, "debug_conv: cond_ld < Cout");
      REQUIRE(q.res >= 0 && q.res <= 2 && (q.res != 1 || res) && (q.res != 2 || q.y_on), VTTS_ERR_INVALID, "debug_conv: bad residual");
      REQUIRE(q.y_on || q.planes_on, VTTS_ERR_INVALID, "debug_conv: a problem must write y or planes");
      if (q.planes_on) {
        REQUIRE(p_out && (p_planes == 2 || p_planes == 3) && q.ldp > 0 && q.poff >= 0, VTTS_ERR_INVALID, "debug_conv: bad output planes");
        any_planes = true;
      }
      if (q.y_on) REQUIRE(y && q.ldy > 0 && q.yoff >= 0, VTTS_ERR_INVALID, "debug_conv: bad y");
      if (use_tc) {
        REQUIRE(q.Cin % TC_BK == 0 && q.Cin == P0.Cin && q.in_extra == P0.in_extra, VTTS_ERR_INVALID,
                "debug_conv: tensor-core problems share one input of Cin (a multiple of 64) channels and in_extra rows");
        REQUIRE(q.w_hi && q.w_lo && (x_planes == 3) == (q.w_mid != nullptr), VTTS_ERR_INVALID,
                "debug_conv: mixed plane counts (every problem's weights must have as many planes as the input)");
        REQUIRE(!q.reflect && !q.pro && q.ldx == 0 && q.xoff == 0, VTTS_ERR_INVALID, "debug_conv: reflect / prologue / ldx are FFMA-only");
        REQUIRE(!q.planes_on || q.ldp >= q.poff + ((q.epi & TCE_GATE) ? q.Cout / 2 : q.Cout), VTTS_ERR_INVALID, "debug_conv: ldp too small");
      } else {
        REQUIRE(q.Cin % CV_CK == 0, VTTS_ERR_INVALID, "debug_conv: FFMA input channels must be a multiple of 16");
        REQUIRE(q.w && q.y_on && q.poff == 0 && q.pro >= 0 && q.pro <= 1, VTTS_ERR_INVALID, "debug_conv: the FFMA conv writes y, takes w and no poff");
        REQUIRE(q.ldx % 4 == 0 && q.xoff % 4 == 0 && q.ldx >= q.xoff + q.Cin, VTTS_ERR_INVALID, "debug_conv: FFMA input rows are read as float4");
        REQUIRE(CV_TT + (q.k - 1) * q.dil <= 32 * CV_XR, VTTS_ERR_INVALID, "debug_conv: halo larger than the FFMA tile");
        REQUIRE(!q.reflect || (q.in_extra == 1 && q.pad == 0), VTTS_ERR_INVALID, "debug_conv: reflect maps ReflectionPad1d((1,0)) (in_extra 1, pad 0)");
      }
    }
    // rows written per utterance must fit the buffers; inputs must cover every utterance's rows
    auto check_rows = [&](size_t n, int ld, int col0, int ncol, const vtts_conv_problem& q, const char* what) {
      for (int b = 0; b < B; ++b) {
        const long L = (long)lens[b] * rmul + q.in_extra;
        const long last = off[b] * rmul * q.out_mul + (long)b * q.out_seq_extra + (L - 1) * q.out_mul + q.out_add;
        REQUIRE((size_t)(last * ld + col0 + ncol) <= n, VTTS_ERR_INVALID, std::string("debug_conv: ") + what + " buffer too small");
      }
    };
    for (int i = 0; i < n_problems; ++i) {
      const vtts_conv_problem& q = problems[i];
      const int ncol = (q.epi & EPI_GATE) ? q.Cout / 2 : q.Cout;
      if (q.y_on) check_rows(y_n, q.ldy, q.yoff, ncol, q, "y");
      if (q.res == 1) check_rows(res_n, q.ldr, q.roff, ncol, q, "res");
      if (q.res == 2) check_rows(y_n, q.ldr, q.roff, ncol, q, "residual (y)");
      if (q.planes_on) check_rows(p_n, q.ldp, q.poff, ncol, q, "planes");
      if (!use_tc) {
        for (int b = 0; b < B; ++b) {
          const long Lp = (long)lens[b] * rmul;
          REQUIRE(!q.reflect || Lp >= 2, VTTS_ERR_INVALID, "debug_conv: reflect needs >= 2 input rows per utterance");
          const long lastrow = off[b] * rmul + (q.reflect ? Lp - 1 : Lp + q.in_extra - 1);
          REQUIRE((size_t)(lastrow * q.ldx + q.xoff + q.Cin) <= x_n, VTTS_ERR_INVALID, "debug_conv: x buffer too small");
        }
      }
    }
    // tensor cores: the input planes as a phase holds them (rows behind each utterance read as zero through the zeroed tails,
    // TMA's out-of-bounds fill in front of the first and behind the last row) -- the halo must stay inside that
    const int extra = P0.in_extra;
    const long end_last = (off[B - 1] + lens[B - 1]) * rmul + (long)B * extra;
    const long units = use_tc ? std::max<long>(off[B], ((long)x_n - (long)B * extra + rmul - 1) / rmul) : 0;
    const long rows_cap = units * rmul + (long)B * extra;
    if (use_tc) {
      REQUIRE((long)x_n >= end_last, VTTS_ERR_INVALID, "debug_conv: x planes have fewer rows than the packed utterances");
      const long inner = gap <= 2 * ZT_ROWS ? gap : ZT_ROWS;          // zeroed rows between two utterances (zero_tails_kernel)
      for (int i = 0; i < n_problems; ++i) {
        const vtts_conv_problem& q = problems[i];
        const long left = q.pad, right = (long)(q.k - 1) * q.dil - q.pad;
        REQUIRE(B == 1 || (left <= inner && right <= inner), VTTS_ERR_INVALID, "debug_conv: conv halo wider than the zeroed gap between utterances");
        REQUIRE(right <= ZT_ROWS || rows_cap <= end_last + ZT_ROWS, VTTS_ERR_INVALID, "debug_conv: conv halo reaches rows behind the zeroed tail");
      }
    }
    // planes() and flush_tails() read the member B: restored on every exit
    struct KeepB { vtts_engine* h; int B; ~KeepB() { h->B = B; } } keep{h, h->B};
    h->B = B;
    // ---- device copies (freed on every exit)
    std::vector<Buf<char>> dev;
    cudaStream_t st = h->stream;
    CK(cudaStreamSynchronize(st));
    std::vector<int> lo(2 * B + 1);
    for (int b = 0; b < B; ++b) lo[b] = lens[b];
    for (int b = 0; b <= B; ++b) lo[B + b] = (int)off[b];
    int* dl = static_cast<int*>(upload(dev, lo.data(), lo.size() * sizeof(int), st));
    const int* dlens = dl;
    const int* doffs = dl + B;
    const std::vector<int> hl(lens, lens + B);     // the heuristics see this call's lengths
    const Rows r{dlens, doffs, B, maxLen, hl, hl, ov ? h->tune.with(*ov) : h->tune};
    float* dy = y ? static_cast<float*>(upload(dev, y, y_n * sizeof(float), st)) : nullptr;
    const float* dres = res ? static_cast<const float*>(upload(dev, res, res_n * sizeof(float), st)) : nullptr;
    __nv_bfloat16* dp = any_planes ? static_cast<__nv_bfloat16*>(upload(dev, p_out, (size_t)p_planes * p_n * 2, st)) : nullptr;
    __nv_bfloat16 *dp_hi = dp, *dp_mid = (dp && p_planes == 3) ? dp + p_n : nullptr, *dp_lo = dp ? dp + (p_planes - 1) * p_n : nullptr;
    auto cond_of = [&](const vtts_conv_problem& q) {
      return q.cond ? static_cast<const float*>(upload(dev, q.cond, (size_t)B * q.cond_ld * sizeof(float), st)) : nullptr;
    };
    if (use_tc) {
      const int Cin = P0.Cin;
      h->begin_planes();
      Planes in = h->planes(57, units, rmul, Cin, extra, x_planes == 3);
      const uint16_t* xs = static_cast<const uint16_t*>(x);
      __nv_bfloat16* dst[3] = {in.hi, x_planes == 3 ? in.mid : in.lo, in.lo};
      for (int pl = 0; pl < x_planes; ++pl)
        CK(cudaMemcpyAsync(dst[pl], xs + (size_t)pl * x_n * Cin, x_n * Cin * 2, cudaMemcpyHostToDevice, st));
      h->flush_tails(dlens, doffs);
      std::vector<TcSpec> ps;
      for (int i = 0; i < n_problems; ++i) {
        const vtts_conv_problem& q = problems[i];
        const size_t wn = (size_t)q.k * q.Cout * q.Cin;
        TcSpec s;
        s.in = in;
        s.w.hi = static_cast<const __nv_bfloat16*>(upload(dev, q.w_hi, wn * 2, st));
        s.w.lo = static_cast<const __nv_bfloat16*>(upload(dev, q.w_lo, wn * 2, st));
        if (q.w_mid) s.w.mid = static_cast<const __nv_bfloat16*>(upload(dev, q.w_mid, wn * 2, st));
        s.bias = static_cast<const float*>(upload(dev, q.bias, (size_t)q.Cout * sizeof(float), st));
        s.Cin = q.Cin; s.Cout = q.Cout; s.k = q.k; s.dil = q.dil; s.pad = q.pad;
        s.y = q.y_on ? dy : nullptr; s.ldy = q.ldy; s.yoff = q.yoff;
        s.res = q.res == 1 ? dres : (q.res == 2 ? dy : nullptr); s.ldr = q.ldr; s.roff = q.roff;
        if (q.planes_on) { s.out.hi = dp_hi; s.out.lo = dp_lo; s.out.mid = dp_mid; s.out.C = q.ldp; }
        s.pl_slope = q.pl_slope; s.poff = q.poff;
        s.out_mul = q.out_mul; s.out_add = q.out_add; s.in_extra = q.in_extra; s.out_seq_extra = q.out_seq_extra;
        s.epi = q.epi; s.alpha = q.alpha;
        s.cond = cond_of(q); s.cond_ld = q.cond_ld;
        ps.push_back(s);
      }
      h->launch_tc(ps, rmul, r);
    } else {
      const float* dx = static_cast<const float*>(upload(dev, x, x_n * sizeof(float), st));
      std::vector<ConvP> ps;
      for (int i = 0; i < n_problems; ++i) {
        const vtts_conv_problem& q = problems[i];
        ConvW W;
        W.Cin = q.Cin; W.Cout = q.Cout; W.k = q.k; W.ldw = (q.Cout + 3) / 4 * 4;
        W.w = static_cast<const float*>(upload(dev, q.w, (size_t)q.k * q.Cin * W.ldw * sizeof(float), st));
        W.b = static_cast<const float*>(upload(dev, q.bias, (size_t)W.ldw * sizeof(float), st));
        ConvP p = mk(W, dx, q.ldx, q.xoff, dy, q.ldy, q.yoff, q.dil, q.pad);
        p.cond = cond_of(q); p.cond_ld = q.cond_ld;
        p.res = q.res == 1 ? dres : (q.res == 2 ? dy : nullptr); p.ldr = q.ldr; p.roff = q.roff;
        p.in_extra = q.in_extra; p.reflect = q.reflect; p.out_mul = q.out_mul; p.out_add = q.out_add; p.out_seq_extra = q.out_seq_extra;
        p.pro = q.pro; p.slope = q.slope; p.epi = q.epi; p.alpha = q.alpha;
        if (q.planes_on) { p.p_hi = dp_hi; p.p_lo = dp_lo; p.p_mid = dp_mid; p.ldp = q.ldp; }
        p.pl_slope = q.pl_slope;
        ps.push_back(p);
      }
      h->launch_conv(ps, rmul, r);
    }
    CK(cudaStreamSynchronize(st));
    if (y) CK(cudaMemcpy(y, dy, y_n * sizeof(float), cudaMemcpyDeviceToHost));
    if (dp) CK(cudaMemcpy(p_out, dp, (size_t)p_planes * p_n * 2, cudaMemcpyDeviceToHost));
    if (report) *report = h->last_conv;
  });
}

int vtts_debug_conv_log(vtts_handle h, int mode, vtts_conv_report* out, int max_n, int* n_out) {
  return guarded(h, [&] {
    REQUIRE(mode >= 0 && mode <= 2, VTTS_ERR_INVALID, "debug_conv_log: mode 0, 1 or 2");
    if (mode == 1) { h->conv_log.clear(); h->log_conv = true; }
    else if (mode == 0) h->log_conv = false;
    else {
      REQUIRE(out && n_out && max_n >= 0, VTTS_ERR_INVALID, "debug_conv_log: missing output");
      const int n = std::min<int>(max_n, (int)h->conv_log.size());
      std::copy(h->conv_log.begin(), h->conv_log.begin() + n, out);
      *n_out = n;
    }
  }, G_ATOMIC, ANY_FAMILY);
}

// ---- Unit-test hooks of the duration path (include/vtts.h): the kernels' own launches on host tensors.
namespace {

// Utterances of the duration hooks packed as the engine packs them (pack_rows), checked against the caller's row count;
// `dev` receives their device copy [lens B][offs B + 1].
struct HookRows {
  std::vector<int> len, off;
  int maxLen = 0;
  int* d = nullptr;
  const int* lens() const { return d; }
  const int* offs() const { return d + len.size(); }
};
HookRows hook_rows(const char* who, int B, const int* lens, size_t rows) {
  REQUIRE(lens && B >= 1 && B <= 16384, VTTS_ERR_INVALID, std::string(who) + ": bad batch size or missing lengths");
  HookRows hr;
  hr.len.assign(lens, lens + B);
  for (int b = 0; b < B; ++b) {
    REQUIRE(lens[b] >= 1, VTTS_ERR_INVALID, std::string(who) + ": lengths must be >= 1");
    hr.maxLen = std::max(hr.maxLen, lens[b]);
  }
  vtts_engine::pack_rows(hr.len, hr.off);
  REQUIRE(rows >= (size_t)hr.off[B], VTTS_ERR_INVALID, std::string(who) + ": fewer rows than the packed utterances");
  return hr;
}
void upload_rows(HookRows& hr, std::vector<Buf<char>>& dev, cudaStream_t st) {
  std::vector<int> lo(hr.len);
  lo.insert(lo.end(), hr.off.begin(), hr.off.end());
  hr.d = static_cast<int*>(upload(dev, lo.data(), lo.size() * sizeof(int), st));
}

}  // namespace

int vtts_debug_dds(vtts_handle h, const char* stack, int B, const int* lens, size_t rows, const float* x, const float* x0,
                   const float* cond, float* y) {
  return guarded(h, [&] {
    REQUIRE(stack && y, VTTS_ERR_INVALID, "debug_dds: missing stack or output");
    const vtts_config& c = h->cfg;
    const int D = c.dp_filter_channels;
    const std::string nm(stack);
    const DdsW* d = nullptr;
    const CfW* F = nullptr;
    if (nm == "dp.convs") {
      d = h->dp_dds;
    } else if (nm.rfind("dp.flows.", 0) == 0 && nm.size() > 15 && nm.compare(nm.size() - 6, 6, ".convs") == 0) {
      // the reference's module index: the ConvFlow n (2 .. dp_n_flows) is dp.flows.<2n - 1>
      const std::string idx = nm.substr(9, nm.size() - 15);
      REQUIRE(idx.size() <= 3 && idx.find_first_not_of("0123456789") == std::string::npos, VTTS_ERR_INVALID,
              "debug_dds: stack must be dp.convs or dp.flows.<2n-1>.convs");
      const int i = atoi(idx.c_str()), n = (i + 1) / 2;
      REQUIRE(i % 2 == 1 && n >= 2 && n <= c.dp_n_flows, VTTS_ERR_INVALID, "debug_dds: no such ConvFlow");
      F = &h->cf[n - 2];
      d = F->dds;
    }
    REQUIRE(d != nullptr, VTTS_ERR_INVALID, "debug_dds: stack must be dp.convs or dp.flows.<2n-1>.convs");
    REQUIRE(F ? (x0 && cond && !x) : (x && !x0 && !cond), VTTS_ERR_INVALID,
            "debug_dds: dp.convs takes x, a ConvFlow stack takes x0 and cond");
    HookRows hr = hook_rows("debug_dds", B, lens, rows);
    std::vector<Buf<char>> dev;
    cudaStream_t st = h->stream;
    CK(cudaStreamSynchronize(st));
    upload_rows(hr, dev, st);
    const size_t n = rows * D;
    // the layers of dds_stack, each into its own buffer holding the caller's rows, so that every layer can be checked on
    // the kernel's own input
    const float* in = static_cast<const float*>(upload(dev, x, n * sizeof(float), st));
    float* out = static_cast<float*>(upload(dev, y, 3 * n * sizeof(float), st));
    const float* dx0 = F ? static_cast<const float*>(upload(dev, x0, rows * sizeof(float), st)) : nullptr;
    const float* dc = F ? static_cast<const float*>(upload(dev, cond, n * sizeof(float), st)) : nullptr;
    const Rows r{hr.lens(), hr.offs(), B, hr.maxLen, hr.len, hr.len, h->tune};
    for (int i = 0, dil = 1; i < 3; ++i, dil *= c.dp_kernel_size) {
      h->dds_layer(d[i], D, c.dp_kernel_size, dil, in, out + i * n, r, i == 0 ? dx0 : nullptr, F ? F->pre_w : nullptr,
                   F ? F->pre_b : nullptr, dc);
      in = out + i * n;
    }
    CK(cudaStreamSynchronize(st));
    CK(cudaMemcpy(y, out, 3 * n * sizeof(float), cudaMemcpyDeviceToHost));
  });
}

int vtts_debug_spline(vtts_handle h, int B, const int* lens, size_t rows, const float* params, int ldh, float* x1) {
  return guarded(h, [&] {
    const vtts_config& c = h->cfg;
    REQUIRE(params && x1, VTTS_ERR_INVALID, "debug_spline: missing parameters or x1");
    REQUIRE(ldh >= 3 * c.dp_num_bins - 1, VTTS_ERR_INVALID, "debug_spline: parameter rows narrower than 3 * dp_num_bins - 1");
    HookRows hr = hook_rows("debug_spline", B, lens, rows);
    std::vector<Buf<char>> dev;
    cudaStream_t st = h->stream;
    CK(cudaStreamSynchronize(st));
    upload_rows(hr, dev, st);
    const float* dp = static_cast<const float*>(upload(dev, params, rows * ldh * sizeof(float), st));
    float* dx = static_cast<float*>(upload(dev, x1, rows * sizeof(float), st));
    h->klaunch(spline_inverse_kernel, dim3((hr.maxLen + 127) / 128, B), dim3(128), (size_t)0, dp, ldh, dx, c.dp_num_bins, c.dp_tail_bound,
               sqrtf((float)c.dp_filter_channels), hr.lens(), hr.offs());
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    CK(cudaMemcpy(x1, dx, rows * sizeof(float), cudaMemcpyDeviceToHost));
  });
}

int vtts_debug_t2s_sample(vtts_handle h, int B, const float* logits, int32_t* state, int32_t* y, int y_ld, int top_k, float top_p,
                          float temperature, float penalty, int early_stop, int step_cap, const uint64_t* seeds, const float* q, int q_ld,
                          uint32_t* seen, int32_t* n_stopped, float* raw, int raw_ld) {
  return guarded(h, [&] {
    const int V = h->t2s_vocab, nw = (V + 31) / 32;
    REQUIRE(B >= 1 && B <= 4096, VTTS_ERR_INVALID, "debug_t2s_sample: bad batch size");
    REQUIRE(logits && state && y && seen && n_stopped, VTTS_ERR_INVALID, "debug_t2s_sample: missing input or output");
    REQUIRE(!q != !seeds, VTTS_ERR_INVALID, "debug_t2s_sample: give per-row seeds or q, not both");
    REQUIRE(top_k >= 1 && std::isfinite(top_p) && std::isfinite(temperature) && std::isfinite(penalty) && penalty > 0.f &&
                early_stop >= -1 && step_cap >= 1,
            VTTS_ERR_INVALID, "debug_t2s_sample: bad sampling arguments");
    REQUIRE(!raw || raw_ld >= 1, VTTS_ERR_INVALID, "debug_t2s_sample: raw_ld must be >= 1");
    REQUIRE(y_ld >= 1 && (size_t)B * y_ld < (1u << 31), VTTS_ERR_INVALID, "debug_t2s_sample: y_ld must be >= 1 and y below 2^31 slots");
    // each row's tokens sit at y[b][0 ..): its state's YOFF is b * y_ld, and its previous tokens y[b][0, P + GEN) mark the
    // seen bitmap, as t2s_init_kernel and the earlier steps leave it
    std::vector<int32_t> sh(state, state + (size_t)B * T2S_ST);
    std::vector<uint32_t> sn((size_t)B * nw, 0u);
    for (int b = 0; b < B; ++b) {
      int32_t* s = sh.data() + (size_t)b * T2S_ST;
      const int P = s[ST_P], gen = s[ST_GEN], ny = s[ST_NY];
      REQUIRE(P >= 0 && gen >= 0 && ny >= 0 && ny <= P + gen && (s[ST_STOP] == 0 || s[ST_STOP] == 1), VTTS_ERR_INVALID,
              "debug_t2s_sample: a row's state is out of range (P, GEN >= 0, 0 <= NY <= P + GEN, STOP 0 or 1)");
      REQUIRE(y_ld > P + gen, VTTS_ERR_INVALID, "debug_t2s_sample: y_ld must exceed P + GEN, the slot of the next token");
      REQUIRE(!q || q_ld > gen, VTTS_ERR_INVALID, "debug_t2s_sample: q_ld must exceed GEN, the row of this step's draws");
      s[ST_YOFF] = b * y_ld;
      for (int i = 0; i < P + gen; ++i) {
        const int tok = y[(size_t)b * y_ld + i];
        REQUIRE(tok >= 0 && tok < V, VTTS_ERR_INVALID, "debug_t2s_sample: a previous token is outside the vocabulary");
        sn[(size_t)b * nw + (tok >> 5)] |= 1u << (tok & 31);
      }
    }
    std::vector<Buf<char>> dev;
    cudaStream_t st = h->stream;
    CK(cudaStreamSynchronize(st));
    const T2sPrm prm{top_p, temperature, penalty, top_k, early_stop, step_cap, q ? q_ld : 0, raw ? raw_ld : 0};
    const float* dlg = static_cast<const float*>(upload(dev, logits, (size_t)B * V * sizeof(float), st));
    const T2sPrm* dprm = static_cast<const T2sPrm*>(upload(dev, &prm, sizeof(prm), st));
    const unsigned long long* dsd = seeds ? static_cast<const unsigned long long*>(upload(dev, seeds, (size_t)B * 8, st)) : nullptr;
    const float* dq = q ? static_cast<const float*>(upload(dev, q, (size_t)B * q_ld * V * sizeof(float), st)) : nullptr;
    float* draw = raw ? static_cast<float*>(upload(dev, raw, (size_t)B * raw_ld * V * sizeof(float), st)) : nullptr;
    int* dst = static_cast<int*>(upload(dev, sh.data(), sh.size() * sizeof(int), st));
    int* dy = static_cast<int*>(upload(dev, y, (size_t)B * y_ld * sizeof(int), st));
    unsigned* dsn = static_cast<unsigned*>(upload(dev, sn.data(), sn.size() * sizeof(unsigned), st));
    const int zero = 0;
    int* dns = static_cast<int*>(upload(dev, &zero, sizeof(int), st));
    h->klaunch(t2s_sample_kernel, dim3(B), dim3(T2S_SAMPLE_THREADS), (size_t)0, dlg, dprm, dsd, dq, draw, dst, dy, dsn, dns, V);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    CK(cudaMemcpy(state, dst, (size_t)B * T2S_ST * sizeof(int), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(y, dy, (size_t)B * y_ld * sizeof(int), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(seen, dsn, sn.size() * sizeof(unsigned), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(n_stopped, dns, sizeof(int), cudaMemcpyDeviceToHost));
    if (raw) CK(cudaMemcpy(raw, draw, (size_t)B * raw_ld * V * sizeof(float), cudaMemcpyDeviceToHost));
  }, G_ATOMIC, VTTS_FAMILY_T2S);
}

int vtts_debug_durations(vtts_handle h, int B, const int* lens, size_t rows, const float* z, float length_scale, int frame_cap,
                         const float* stats, const float* eps, int64_t eps_ld, float noise_scale, int32_t* wceil, int32_t* cum,
                         int32_t* ylen, int32_t* ylen_real, int32_t* frm_off, int32_t* published, size_t frame_rows, float* z_p,
                         int32_t* frame_token) {
  return guarded(h, [&] {
    REQUIRE(z && stats && eps && wceil && cum && ylen && ylen_real && frm_off && published && z_p && frame_token, VTTS_ERR_INVALID,
            "debug_durations: missing input or output");
    REQUIRE(frame_cap >= 0 && eps_ld >= 1, VTTS_ERR_INVALID, "debug_durations: frame_cap must be >= 0 and eps_ld >= 1");
    HookRows hr = hook_rows("debug_durations", B, lens, rows);
    const int I = h->cfg.inter_channels;
    std::vector<Buf<char>> dev;
    cudaStream_t st = h->stream;
    CK(cudaStreamSynchronize(st));
    upload_rows(hr, dev, st);
    float prm[8] = {noise_scale, length_scale, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const int seq = 1;
    memcpy(&prm[6], &seq, 4);
    memcpy(&prm[7], &frame_cap, 4);
    const float* dprm = static_cast<const float*>(upload(dev, prm, sizeof(prm), st));
    const float* dz = static_cast<const float*>(upload(dev, z, rows * sizeof(float), st));
    int* dwc = static_cast<int*>(upload(dev, wceil, rows * sizeof(int), st));
    int* dcum = static_cast<int*>(upload(dev, cum, rows * sizeof(int), st));
    int* dlen = static_cast<int*>(upload(dev, nullptr, (3 * (size_t)B + 1) * sizeof(int), st));   // ylen | ylen_real | offsets
    MappedBuf<int> pub;
    CK(pub.alloc(2 * (size_t)B + 2));
    pub.p[0] = 0;
    // the engine's own ticket counter: it must be back at 0 after every launch
    unsigned int* dctr = reinterpret_cast<unsigned int*>(h->ensure(h->d_done_ctr, 4));
    h->klaunch(duration_kernel, dim3(B), dim3(256), (size_t)0, dz, h->dp_ea, 0, 2, dprm, dwc, dcum, dlen, hr.lens(), hr.offs(),
               dlen + 2 * B, B, (volatile int*)pub.d, dctr, dlen + B);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    REQUIRE(pub.p[0] == seq, VTTS_ERR_CUDA, "debug_durations: the lengths were not published");
    CK(cudaMemcpy(wceil, dwc, rows * sizeof(int), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(cum, dcum, rows * sizeof(int), cudaMemcpyDeviceToHost));
    std::vector<int> lo(3 * B + 1);
    CK(cudaMemcpy(lo.data(), dlen, lo.size() * sizeof(int), cudaMemcpyDeviceToHost));
    std::copy(lo.begin(), lo.begin() + B, ylen);
    std::copy(lo.begin() + B, lo.begin() + 2 * B, ylen_real);
    std::copy(lo.begin() + 2 * B, lo.end(), frm_off);
    std::copy(pub.p + 1, pub.p + 2 * B + 2, published);
    // what the host reads, refused as the engine refuses it; then the prior over the device lengths, as phase 2 runs it
    vtts_engine::check_frame_lengths(pub.p + 1, pub.p[2 * B + 1], B);
    int maxFrm = 0;
    for (int b = 0; b < B; ++b) maxFrm = std::max(maxFrm, lo[b]);
    REQUIRE((size_t)lo[3 * B] <= frame_rows, VTTS_ERR_CAPACITY, "debug_durations: fewer frame rows than the packed frames");
    REQUIRE(eps_ld >= maxFrm, VTTS_ERR_CAPACITY, "debug_durations: eps_ld is smaller than the longest utterance's frames");
    const float* dst = static_cast<const float*>(upload(dev, stats, (size_t)hr.off[B] * 2 * I * sizeof(float), st));
    const float* deps = static_cast<const float*>(upload(dev, eps, (size_t)B * I * eps_ld * sizeof(float), st));
    float* dzp = static_cast<float*>(upload(dev, z_p, frame_rows * I * sizeof(float), st));
    int* dft = static_cast<int*>(upload(dev, frame_token, frame_rows * sizeof(int), st));
    h->klaunch(sample_prior_kernel, dim3(maxFrm, B), dim3(64), (size_t)0, dst, I, (const int*)dcum, hr.lens(), hr.offs(),
               (const int*)dlen, (const int*)(dlen + 2 * B), deps, (int)eps_ld, dprm, dzp, dft);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    CK(cudaMemcpy(z_p, dzp, frame_rows * I * sizeof(float), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(frame_token, dft, frame_rows * sizeof(int), cudaMemcpyDeviceToHost));
  });
}

int vtts_debug_stt_durations(vtts_handle h, int B, const int* lens, size_t rows, const float* mu_dp, const float* pause,
                             float length_scale, const float* x, const float* mu_mel, int denormalise, int32_t* dur, int32_t* first,
                             int32_t* ylen, float* logw, size_t frame_rows, float* mu, float* pau, float* prior, float* mel) {
  return guarded(h, [&] {
    const vtts_config& c = h->cfg;
    REQUIRE(h->st_text, VTTS_ERR_INVALID, "debug_stt_durations: the engine has no text encoder");
    REQUIRE(mu_dp && pause && x && dur && first && ylen && logw && mu && pau && mel, VTTS_ERR_INVALID,
            "debug_stt_durations: missing input or output");
    REQUIRE(!prior || mu_mel, VTTS_ERR_INVALID, "debug_stt_durations: the prior rows need mu_mel");
    HookRows hr = hook_rows("debug_stt_durations", B, lens, rows);
    const int DC = c.st_dur_channels, MC = c.st_cond, NC = c.st_noise;
    std::vector<Buf<char>> dev;
    cudaStream_t st = h->stream;
    CK(cudaStreamSynchronize(st));
    upload_rows(hr, dev, st);
    float prm[16] = {length_scale, 0.f, denormalise ? 1.f : 0.f};
    const float* dprm = static_cast<const float*>(upload(dev, prm, sizeof(prm), st));
    const float* dmu = static_cast<const float*>(upload(dev, mu_dp, rows * DC * sizeof(float), st));
    const float* dpause = static_cast<const float*>(upload(dev, pause, rows * sizeof(float), st));
    int* ddur = static_cast<int*>(upload(dev, dur, rows * sizeof(int), st));
    int* dfirst = static_cast<int*>(upload(dev, first, rows * sizeof(int), st));
    float* dlogw = static_cast<float*>(upload(dev, logw, rows * sizeof(float), st));
    int* dylen = static_cast<int*>(upload(dev, nullptr, (size_t)B * sizeof(int), st));
    h->klaunch(stt_dur_kernel, dim3(B), dim3(STT_SCAN), (size_t)0, dmu, DC, DC, dpause, dprm, (float)VTTS_ST_MAX_TOKEN_FRAMES, ddur, dfirst,
               dylen, dlogw, hr.lens(), hr.offs());
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    CK(cudaMemcpy(dur, ddur, rows * sizeof(int), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(first, dfirst, rows * sizeof(int), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(logw, dlogw, rows * sizeof(float), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(ylen, dylen, (size_t)B * sizeof(int), cudaMemcpyDeviceToHost));
    // frame rows of the utterances, packed as the mel phase packs them
    HookRows fr;
    fr.len.assign(ylen, ylen + B);
    for (int b = 0; b < B; ++b) fr.maxLen = std::max(fr.maxLen, ylen[b]);
    vtts_engine::pack_rows(fr.len, fr.off);
    REQUIRE((size_t)fr.off[B] <= frame_rows, VTTS_ERR_CAPACITY, "debug_stt_durations: fewer frame rows than the packed frames");
    upload_rows(fr, dev, st);
    const float* dx = static_cast<const float*>(upload(dev, x, rows * MC * sizeof(float), st));
    const float* dmm = mu_mel ? static_cast<const float*>(upload(dev, mu_mel, rows * NC * sizeof(float), st)) : nullptr;
    float* dmuf = static_cast<float*>(upload(dev, mu, frame_rows * MC * sizeof(float), st));
    float* dpau = static_cast<float*>(upload(dev, pau, frame_rows * sizeof(float), st));
    float* dprior = prior ? static_cast<float*>(upload(dev, prior, frame_rows * NC * sizeof(float), st)) : nullptr;
    float* dmel = static_cast<float*>(upload(dev, mel, frame_rows * NC * sizeof(float), st));
    h->klaunch(stt_expand_kernel, dim3(hr.maxLen, B), dim3(128), (size_t)0, dx, MC, dpause, dmm, NC, (const int*)ddur, (const int*)dfirst,
               dmuf, dpau, dprior, dprm, h->st_mel_mean, h->st_mel_std, hr.lens(), hr.offs(), fr.offs());
    h->klaunch(stt_pause_fill_kernel, dim3(fr.maxLen, B), dim3(128), (size_t)0, dmel, NC, (const float*)dpau, fr.lens(), fr.offs());
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    CK(cudaMemcpy(mu, dmuf, frame_rows * MC * sizeof(float), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(pau, dpau, frame_rows * sizeof(float), cudaMemcpyDeviceToHost));
    if (prior) CK(cudaMemcpy(prior, dprior, frame_rows * NC * sizeof(float), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(mel, dmel, frame_rows * NC * sizeof(float), cudaMemcpyDeviceToHost));
  }, G_ATOMIC, VTTS_FAMILY_STABLETTS);
}

// ---- Unit-test hooks of the spectral kernels (include/vtts.h): the front end and the decoder tail on host tensors.
int vtts_debug_front_end(vtts_handle h, int from_spec, const float* in, const int64_t* lengths, int B, int64_t ld, int32_t* frames,
                         size_t rows, float* mag, float* feat) {
  return guarded(h, [&] {
    const vtts_config& c = h->cfg;
    REQUIRE(h->stft_basis, VTTS_ERR_INVALID, "debug_front_end: the engine has no spectrogram front end");
    REQUIRE(in && lengths && frames && feat, VTTS_ERR_INVALID, "debug_front_end: missing input or output");
    const bool mel = !from_spec && c.use_mel_posterior_encoder;
    REQUIRE(mel == (mag != nullptr), VTTS_ERR_INVALID, "debug_front_end: mag is the magnitude rows of a mel engine's waveform input "
            "(NULL otherwise: a linear engine's magnitude rows are the features)");
    const std::vector<int> fr = clip_frames(h, from_spec != 0, lengths, B, ld);
    std::vector<int> off;
    vtts_engine::pack_rows(fr, off);
    REQUIRE(rows >= (size_t)off[B], VTTS_ERR_INVALID, "debug_front_end: fewer rows than the packed frames");
    const size_t nbins = c.filter_length / 2 + 1, n = off[B];
    h->B = B;
    h->have_durations = false;
    h->have_latent = false;
    stage_clips(h, from_spec != 0, in, lengths, ld, fr, nullptr, nullptr, 0.f, nullptr, 0, 0);
    if (!from_spec) {     // NaN behind every clip in the staging, so that a read outside a clip shows in its rows
      float* pin = h->stg[vtts_engine::STG_CLIPS].host(h->d_vin);
      for (int b = 0; b < B; ++b)
        std::fill(pin + (size_t)b * h->vc_wld + lengths[b], pin + (size_t)(b + 1) * h->vc_wld, std::nanf(""));
    }
    cudaStream_t st = h->stream;
    h->vc_upload(false);
    float* dfeat = h->ensure(h->d_vfeat, (size_t)h->Tfrm * h->spec_pad);
    float* dmag = mel ? h->ensure(h->d_vlin, (size_t)h->Tfrm * nbins) : nullptr;
    CK(cudaMemcpyAsync(dfeat, feat, n * h->spec_pad * sizeof(float), cudaMemcpyHostToDevice, st));
    if (mel) CK(cudaMemcpyAsync(dmag, mag, n * nbins * sizeof(float), cudaMemcpyHostToDevice, st));
    REQUIRE(h->front_end(from_spec != 0) == dfeat, VTTS_ERR_CUDA, "debug_front_end: the front end wrote another buffer");
    CK(cudaStreamSynchronize(st));
    CK(cudaMemcpy(feat, dfeat, n * h->spec_pad * sizeof(float), cudaMemcpyDeviceToHost));
    if (mel) CK(cudaMemcpy(mag, dmag, n * nbins * sizeof(float), cudaMemcpyDeviceToHost));
    std::copy(fr.begin(), fr.end(), frames);
  }, G_ATOMIC, ANY_FAMILY);
}

int vtts_debug_istft(vtts_handle h, int B, const int* lens, int first, size_t rows, const float* post, size_t n_wav, float* wav) {
  return guarded(h, [&] {
    const vtts_config& c = h->cfg;
    REQUIRE(h->istft_basis && h->pqmf, VTTS_ERR_INVALID, "debug_istft: the engine has no inverse-STFT decoder");
    REQUIRE(post && wav, VTTS_ERR_INVALID, "debug_istft: missing input or output");
    REQUIRE(first >= 0, VTTS_ERR_INVALID, "debug_istft: first must be >= 0");
    HookRows hr = hook_rows("debug_istft", B, lens, (size_t)-1);
    for (int& o : hr.off) {
      REQUIRE((int64_t)o + first < (1LL << 30), VTTS_ERR_INVALID, "debug_istft: first row too large");
      o += first;
    }
    const int rm = h->up_total, pc = c.subbands * (c.istft_n_fft + 2);
    REQUIRE(rows >= (size_t)hr.off[B] * rm + B, VTTS_ERR_INVALID, "debug_istft: fewer post rows than the packed utterances' frames");
    REQUIRE(n_wav >= (size_t)hr.off[B] * h->hop, VTTS_ERR_INVALID, "debug_istft: fewer samples than the packed utterances'");
    std::vector<Buf<char>> dev;
    cudaStream_t st = h->stream;
    CK(cudaStreamSynchronize(st));
    upload_rows(hr, dev, st);
    const float* dpost = static_cast<const float*>(upload(dev, post, rows * pc * sizeof(float), st));
    float* dwav = static_cast<float*>(upload(dev, wav, n_wav * sizeof(float), st));
    const Rows r{hr.lens(), hr.offs(), B, hr.maxLen, hr.len, hr.len, h->tune};
    h->istft_tail(dpost, rm, r, dwav);
    CK(cudaStreamSynchronize(st));
    CK(cudaMemcpy(wav, dwav, n_wav * sizeof(float), cudaMemcpyDeviceToHost));
  }, G_ATOMIC, ANY_FAMILY);
}

int vtts_debug_mrf_mean(vtts_handle h, int use_tc, int B, const int* lens, int rmul, int C, int n, size_t rows, const float* x,
                        int last, float* out, size_t plane_rows, uint16_t* hi, uint16_t* lo) {
  return guarded(h, [&] {
    REQUIRE(x && (use_tc ? (hi && lo) : (out && !hi && !lo)), VTTS_ERR_INVALID,
            "debug_mrf_mean: x and out (FFMA), or x, hi and lo (tensor cores) are required");
    REQUIRE(n >= 1 && n <= 3 && C >= 4 && C % 4 == 0 && rmul >= 1, VTTS_ERR_INVALID,
            "debug_mrf_mean: needs 1 to 3 inputs, C a multiple of 4 and rmul >= 1");
    HookRows hr = hook_rows("debug_mrf_mean", B, lens, (size_t)-1);
    REQUIRE(rows >= (size_t)hr.off[B] * rmul, VTTS_ERR_INVALID, "debug_mrf_mean: fewer rows than the packed utterances'");
    if (use_tc) {
      REQUIRE(plane_rows >= (size_t)hr.off[B] * rmul + (last ? B : 0), VTTS_ERR_INVALID,
              "debug_mrf_mean: fewer plane rows than the packed utterances' (and their reflect rows)");
      for (int b = 0; b < B; ++b)
        REQUIRE(!last || (int64_t)lens[b] * rmul >= 2, VTTS_ERR_INVALID, "debug_mrf_mean: the reflect row needs 2 rows per utterance");
    }
    std::vector<Buf<char>> dev;
    cudaStream_t st = h->stream;
    CK(cudaStreamSynchronize(st));
    upload_rows(hr, dev, st);
    const size_t nx = rows * C;
    const float* dx = static_cast<const float*>(upload(dev, x, n * nx * sizeof(float), st));
    std::vector<float*> xj;
    for (int j = 0; j < n; ++j) xj.push_back(const_cast<float*>(dx) + j * nx);
    float* dout = out ? static_cast<float*>(upload(dev, out, nx * sizeof(float), st)) : nullptr;
    Planes pl;
    if (use_tc) {
      pl.hi = static_cast<__nv_bfloat16*>(upload(dev, hi, plane_rows * C * 2, st));
      pl.lo = static_cast<__nv_bfloat16*>(upload(dev, lo, plane_rows * C * 2, st));
      const Rows r{hr.lens(), hr.offs(), B, hr.maxLen, hr.len, hr.len, h->tune};
      h->mrf_mean_planes(xj, dout, pl, C, last != 0, rmul, r);
    } else {
      h->mrf_mean(xj, dout, (long)(nx / 4));
    }
    CK(cudaStreamSynchronize(st));
    if (out) CK(cudaMemcpy(out, dout, nx * sizeof(float), cudaMemcpyDeviceToHost));
    if (use_tc) {
      CK(cudaMemcpy(hi, pl.hi, plane_rows * C * 2, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(lo, pl.lo, plane_rows * C * 2, cudaMemcpyDeviceToHost));
    }
  }, G_ATOMIC, ANY_FAMILY);
}

// Host-only restatement of launch_tc's split-K plan (tc_split_plan) for tests: no device, no engine.
int vtts_tc_split_plan(int n, const int* cin, const int* cout, const int* k, const int* in_extra, int B, const int* lens,
                       int rmul, int max_len, int bn, int max_split, int min_steps, int n_sm, const int* cluster_cap, int* plan) {
  if (n < 1 || n > TC_MAXP || B < 1 || rmul < 1 || max_len < 0 || !cin || !cout || !k || !in_extra || !lens || !cluster_cap || !plan)
    return VTTS_ERR_INVALID;
  if ((bn != 0 && bn != 64 && bn != 128) || max_split < 1 || min_steps < 1 || n_sm < 1) return VTTS_ERR_INVALID;
  TcSplitIn in;
  in.n = n; in.nb = B; in.gx = 0;
  in.bn = bn; in.max_split = max_split; in.min_steps = min_steps; in.n_sm = n_sm;
  memcpy(in.cluster_cap, cluster_cap, sizeof(in.cluster_cap));
  in.lens = lens; in.rmul = rmul;
  for (int p = 0; p < n; ++p) {
    if (cin[p] < TC_BK || cin[p] % TC_BK || k[p] < 1 || cout[p] < 1 || in_extra[p] < 0) return VTTS_ERR_INVALID;
    in.steps[p] = cin[p] / TC_BK * k[p];
    in.cout[p] = cout[p];
    in.in_extra[p] = in_extra[p];
    in.gx = std::max(in.gx, (max_len * rmul + in_extra[p] + TC_BM - 1) / TC_BM);
  }
  for (int b = 0; b < B; ++b)
    if (lens[b] < 0 || lens[b] > max_len) return VTTS_ERR_INVALID;
  const TcSplitPlan pl = tc_split_plan(in);
  plan[0] = pl.bn; plan[1] = pl.split;
  for (int p = 0; p < TC_MAXP; ++p) plan[2 + p] = p < n ? pl.psplit[p] : 0;
  return VTTS_OK;
}

int vtts_profile_read_tc(vtts_handle h, double* ms, uint64_t* launches, double* flops) {
  if (!ms || !launches || !flops) return VTTS_ERR_INVALID;
  return guarded(h, [&] {
    CK(cudaStreamSynchronize(h->stream));
    double t = 0.0;
    for (size_t i = 0; i + 1 < h->tc_prof_used; i += 2) {
      float e = 0.f;
      CK(cudaEventElapsedTime(&e, h->tc_prof_ev[i], h->tc_prof_ev[i + 1]));
      t += e;
    }
    *ms = t;
    *launches = h->tc_prof_launches;
    *flops = h->tc_prof_flops;
  }, G_ATOMIC, ANY_FAMILY);
}

// Micro-benchmark of one conv kernel in isolation (back-to-back launches, CUDA events on the engine stream):
//   what = "tc:<Cin>:<Cout>:<k>:<dil>:<rows>"   wgmma kernel (precision mode 1 engines only)
//          "ffma:<Cin>:<Cout>:<k>:<dil>:<rows>" fp32 FFMA kernel
// Returns the average milliseconds per launch, or a negative status.  Used by bench.py for the roofline of the
// dominant kernel timed alone, and by tools/ for tuning.
float vtts_microbench(vtts_handle h, const char* what, int iters) {
  if (!h || !what || iters < 1) return -1.f;
  float result = -1.f;
  int rc = guarded(h, [&] {
    char kind[16] = {0};
    int Cin = 0, Cout = 0, k = 1, dil = 1, rows = 0;
    REQUIRE(sscanf(what, "%15[a-z]:%d:%d:%d:%d:%d", kind, &Cin, &Cout, &k, &dil, &rows) == 6, VTTS_ERR_INVALID, "bad microbench spec");
    REQUIRE(Cin > 0 && Cout > 0 && k > 0 && rows > 0 && Cin % 64 == 0, VTTS_ERR_INVALID, "bad microbench shape");
    const bool is_tc = strcmp(kind, "tc") == 0;
    REQUIRE(is_tc || strcmp(kind, "ffma") == 0, VTTS_ERR_INVALID, "unknown microbench kind");
    REQUIRE(!is_tc || h->tc, VTTS_ERR_INVALID, "tc microbench needs a precision-1 engine");
    struct KeepProfiling {       // the profiler switch and the stamps buffer, restored on every exit
      vtts_engine* h; bool prof;
      ~KeepProfiling() { h->profiling = prof; h->tc_dbg = nullptr; }
    } keep{h, h->profiling};
    Buf<int> dl, dof;
    Buf<float> x, y, w, bias;
    Buf<__nv_bfloat16> ph, pl, wh, wl;
    const int ldw = (Cout + 3) / 4 * 4;
    CK(dl.alloc(2)); CK(dof.alloc(2));
    const int hl[2] = {rows, rows}, ho[2] = {0, rows};
    CK(cudaMemcpy(dl.p, hl, 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(dof.p, ho, 8, cudaMemcpyHostToDevice));
    const Rows r{dl.p, dof.p, 1, rows, {rows}, {rows}, h->tune};
    CK(y.alloc((size_t)rows * Cout)); CK(bias.alloc(ldw)); CK(cudaMemset(bias.p, 0, (size_t)ldw * 4));
    if (is_tc) {
      CK(ph.alloc((size_t)rows * Cin)); CK(pl.alloc((size_t)rows * Cin));
      CK(wh.alloc((size_t)k * Cout * Cin)); CK(wl.alloc((size_t)k * Cout * Cin));
      CK(cudaMemset(ph.p, 0, (size_t)rows * Cin * 2)); CK(cudaMemset(pl.p, 0, (size_t)rows * Cin * 2));
      CK(cudaMemset(wh.p, 0, (size_t)k * Cout * Cin * 2)); CK(cudaMemset(wl.p, 0, (size_t)k * Cout * Cin * 2));
    } else {
      CK(x.alloc((size_t)rows * Cin)); CK(w.alloc((size_t)k * Cin * ldw));
      CK(cudaMemset(x.p, 0, (size_t)rows * Cin * 4)); CK(cudaMemset(w.p, 0, (size_t)k * Cin * ldw * 4));
    }
    auto once = [&] {
      if (is_tc) {
        TcSpec q;
        q.in.hi = ph.p; q.in.lo = pl.p; q.in.C = Cin; q.in.rows = rows;
        q.w.hi = wh.p; q.w.lo = wl.p; q.bias = bias.p; q.Cin = Cin; q.Cout = Cout; q.k = k; q.dil = dil; q.pad = dil * (k - 1) / 2;
        q.y = y.p; q.ldy = Cout;
        h->launch_tc({q}, 1, r);
      } else {
        ConvW W; W.w = w.p; W.b = bias.p; W.Cin = Cin; W.Cout = Cout; W.k = k; W.ldw = ldw;
        h->launch_conv({mk(W, x.p, Cin, 0, y.p, Cout, 0, dil, dil * (k - 1) / 2)}, 1, r);
      }
    };
    h->profiling = false;
    for (int i = 0; i < 3; ++i) once();
    Event e0, e1;
    CK(cudaEventCreate(e0.out())); CK(cudaEventCreate(e1.out()));
    // the launches are captured into one CUDA graph so that the host launch path is not what gets timed
    Graph graph;
    GraphExec gexec;
    CK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
    for (int i = 0; i < iters; ++i) once();
    CK(cudaStreamEndCapture(h->stream, graph.out()));
    CK(cudaGraphInstantiate(gexec.out(), graph, 0));
    CK(cudaGraphLaunch(gexec, h->stream));           // warm
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaEventRecord(e0, h->stream));
    CK(cudaGraphLaunch(gexec, h->stream));
    CK(cudaEventRecord(e1, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (is_tc && getenv("VTTS_TC_STAMPS")) {
      Buf<unsigned long long> d;
      CK(d.alloc(16)); CK(cudaMemset(d.p, 0, 16 * 8));
      h->tc_dbg = d.p;
      Event a0, a1; CK(cudaEventCreate(a0.out())); CK(cudaEventCreate(a1.out()));
      CK(cudaEventRecord(a0, h->stream));
      once();
      CK(cudaEventRecord(a1, h->stream));
      CK(cudaStreamSynchronize(h->stream));
      h->tc_dbg = nullptr;
      unsigned long long st[16];
      CK(cudaMemcpy(st, d.p, sizeof(st), cudaMemcpyDeviceToHost));
      float one = 0.f; CK(cudaEventElapsedTime(&one, a0, a1));
      fprintf(stderr, "[tc stamps %s] event %.2f us | entry->setup %.2f | ->first TMA issued %.2f | ->all TMA issued %.2f | ->first full %.2f | ->mma issued %.2f | ->acc ready %.2f | ->epi done %.2f | ->sync %.2f (us since entry)\n",
              what, one * 1e3, (st[1] - st[0]) / 1e3, (st[2] - st[0]) / 1e3, (st[3] - st[0]) / 1e3, (st[4] - st[0]) / 1e3,
              (st[5] - st[0]) / 1e3, (st[6] - st[0]) / 1e3, (st[7] - st[0]) / 1e3, (st[8] - st[0]) / 1e3);
    }
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    result = ms / iters;
  });
  return rc == VTTS_OK ? result : (float)rc;
}

}  // extern "C"
