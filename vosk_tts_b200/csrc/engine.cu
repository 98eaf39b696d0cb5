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

template <typename T>
struct Buf {
  T* p = nullptr;
  size_t cap = 0;
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
  vtts_config cfg{};
  int device = 0;
  cudaStream_t stream = nullptr;
  std::mutex mu;
  // The two-phase API (vtts_durations -> vtts_synthesize / vtts_flow) keeps per-handle state between two calls.  A thread
  // that has run vtts_durations owns the handle until its vtts_synthesize / vtts_flow has succeeded (or failed for good);
  // entry points called by OTHER threads wait for that instead of overwriting the pending durations.
  bool two_phase = false;
  std::thread::id owner;
  std::condition_variable cv;
  std::string err;
  uint64_t launches = 0;

  float* d_blob = nullptr;
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
  std::vector<cudaEvent_t> tc_prof_ev;
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
  void assume_frames(int frames) {      // host-side frame shape from a prediction (B == 1)
    h_frm_len.assign(1, frames);
    h_frm_off = {0, frames};
    set_frame_shape();
  }
  bool read_published_lengths() {       // what frame_offsets_kernel wrote into mapped host memory; false: not there (yet)
    if (!h_map || h_map[0] != call_seq) return false;
    h_frm_len.assign(h_map + 1, h_map + 1 + B);
    h_frm_off.assign(h_map + 1 + B, h_map + 1 + 2 * B + 1);
    return true;
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
  Buf<float> d_condv, d_x, d_xb, d_qkv, d_ao, d_y, d_ffh, d_stats, d_dA, d_dB, d_dx, d_h29, d_za, d_zb, d_eps_dp;
  Buf<float> d_z, d_h, d_h1, d_wx, d_acts, d_skip, d_fqkv, d_fao, d_fy, d_ffh2, d_eps_z, d_d0, d_post, d_wav;
  std::vector<Buf<float>> d_stage;               // X_i
  std::vector<std::vector<Buf<float>>> d_xj, d_tmp;
  // per-launch profiling of the conv kernel family (bench.py roofline): event pairs around each launch
  bool profiling = false;
  std::vector<cudaEvent_t> prof_ev;
  size_t prof_used = 0;
  double prof_flops = 0.0;
  uint64_t prof_launches = 0;
  Buf<float> d_zp_dbg;                           // copy of z_p kept when debug_flags & 1
  int debug_flags = 0;
  Buf<char> h_pin, h_pin_in, h_pin_len, h_pin_z;  // pinned staging (host): outputs, phase-1 inputs, lengths, noise_z
  Buf<float> d_prm;                              // per-call scalars (see kernels.cuh prm_seed)
  int* h_map = nullptr;                          // mapped pinned host memory: [0] sequence flag, lengths, offsets
  int* d_map = nullptr;                          // its device alias
  size_t map_cap = 0;
  int call_seq = 0;
  bool use_poll = true;
  // CUDA graphs: a call shape seen before is captured once and replayed (launch-bound at batch 1)
  struct GraphEntry { cudaGraphExec_t exec = nullptr; uint64_t gen = 0; uint64_t used = 0; uint64_t nlaunch = 0; int seen = 0; };
  std::map<std::vector<long long>, GraphEntry> graphs;
  uint64_t ws_gen = 0, graph_clock = 0, graph_replays = 0;
  bool capture_on_first = true;
  bool capturing = false, use_graphs = true, last_graphed = false, use_pdl = true;    // programmatic dependent launch (VTTS_PDL=0 turns it off)
  int conv_max_s = 8, conv_target = 120, conv_max_g = 4, conv_big_g = 1, tc_tall = 0, tc_baseoff = 0, tc_bn = 0, attn_rows = 0, tc_mc = 0, tc_split = 0, conv_min_g = 1, tc_min_steps = 2, conv_auto_g = 4, attn_split = 1, tc_persist = 1, tc_persist_min = 1, n_sm = 132, tc_dbgskip = 0, tc_wmc = 0;
  // shape of the last dense conv launch (vtts_debug_conv) and, while log_conv is set, of every one (vtts_debug_conv_log)
  vtts_conv_report last_conv{};
  vtts_attn_report last_attn{};               // the last attention launch (vtts_debug_attention)
  bool log_conv = false;
  std::vector<vtts_conv_report> conv_log;
  void note_conv(const vtts_conv_report& r) {
    last_conv = r;
    if (log_conv) conv_log.push_back(r);
  }
  int tc_cluster_cap[2][3] = {{0, 0, 0}, {0, 0, 0}};   // co-resident clusters of 2/4/8 conv_tc CTAs, [BN 64/128][log2(S)-1]   // multicast measured slower (see DESIGN.md 4.2)   // tuning knobs (env VTTS_CONV_MAXS / _TARGET / _MAXG)
  cudaEvent_t ev[8] = {};
  cudaStream_t side[3] = {};               // branch streams of the decoder's independent resblock chains (forked / joined with events)
  cudaEvent_t ev_fork = nullptr, ev_join[3] = {};
  int attn_tc_mode = 1;                    // wgmma attention where the qkv conv runs on tensor cores: 0 never, 1 when throughput bound, 2 always
  int mrf_heavy_first = 1;
  int mrf_branch = 0;                      // VTTS_MRF_BRANCH=1: one stream per resblock chain (measured slower: 1.74 vs 1.62 ms)
  float stage_ms[8] = {};
  bool ev_valid = false;

  // -------------------------------------------------------------------------------------------
  template <typename T>
  T* ensure(Buf<T>& b, size_t n) {
    if (n > b.cap) {
      REQUIRE(!capturing, VTTS_ERR_STATE, "workspace growth during graph capture");
      if (b.p) CK(cudaFree(b.p));
      size_t cap = n + n / 4 + 256;
      CK(cudaMalloc(&b.p, cap * sizeof(T)));
      b.cap = cap;
      ++ws_gen;                                // captured graphs hold the old pointers
    }
    return b.p;
  }
  char* ensure_pinned(Buf<char>& hb, size_t n) {
    if (n > hb.cap) {
      REQUIRE(!capturing, VTTS_ERR_STATE, "staging growth during graph capture");
      if (hb.p) {
        CK(cudaStreamSynchronize(stream));   // copies staged through the old buffer may still be in flight
        CK(cudaFreeHost(hb.p));
        hb.p = nullptr;
      }
      size_t cap = n + n / 4 + 4096;
      CK(cudaMallocHost(&hb.p, cap));
      hb.cap = cap;
      ++ws_gen;
    }
    return hb.p;
  }
  char* ensure_pinned(size_t n) { return ensure_pinned(h_pin, n); }

  // Runs `enqueue` (which only enqueues work on `stream`) eagerly the first time a shape key is seen -- that run also
  // performs every workspace growth -- and right behind it records the same work into a CUDA graph (capture only, no second
  // execution), so that the SECOND call of a bucket already replays.  The key is the full tuple of everything the
  // enqueued work depends on besides device-resident data (phase tag, batch, length buckets, noise mode, raw pointers of
  // the *_dev entry points): entries are compared on the tuple itself, so there is no hash collision to replay a wrong
  // graph on.  The cache is bounded (LRU, checked on every insertion).
  static constexpr size_t GRAPH_CACHE_MAX = 48;
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
        if (old->second.exec) cudaGraphExecDestroy(old->second.exec);
        graphs.erase(old);
      }
      it = graphs.emplace(key, GraphEntry{}).first;
    }
    GraphEntry& g = it->second;
    if (g.exec && g.gen != ws_gen) { cudaGraphExecDestroy(g.exec); g.exec = nullptr; g.seen = 0; }
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
    cudaGraph_t graph = nullptr;
    CK(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
    capturing = true;
    try {
      enqueue();
    } catch (...) {
      capturing = false;
      cudaStreamEndCapture(stream, &graph);
      if (graph) cudaGraphDestroy(graph);
      throw;
    }
    capturing = false;
    CK(cudaStreamEndCapture(stream, &graph));
    cudaGraphExec_t exec = nullptr;
    cudaError_t e = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) throw Err{VTTS_ERR_CUDA, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e)};
    g.exec = exec;
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
  bool attn_tc_ok(const EncLayerW& L, int Hc) const;
  bool attn_use_tc(const EncLayerW& L, int Hc, const int* lens, int maxLen) const;
  bool attn_split_fits(const EncLayerW& L, int Hc, const int* lens, int maxLen) const;
  void launch_attn_tc(const Planes& qkv, float* ao, Planes* pl, const EncLayerW& L, int Hc, const int* lens, const int* offs, int maxLen);
  void launch_tc(const std::vector<TcSpec>& ps, int rmul, const int* lens, const int* offs, int maxLen, int nB);
  // plane buffers of the frame-resolution stages: allocated (and their tails zeroed by ONE zero_tails launch) before the
  // first kernel of the phase
  struct FlowPl { Planes ph, pao, ph1, pff, pwx, pacts, pskip, pqkv; } flp;
  struct DecPl { Planes pz, cur; std::vector<Planes> px, nxt; std::vector<std::vector<Planes>> pj, pt; } dcp;
  void alloc_flow_planes();
  void alloc_decoder_planes();
  void decoder_tc(float* z, const int* fl, const int* fo, bool pz_ready);
  void flow_tc(float* z, const int* fl, const int* fo, bool emit_pz, const float* cond, int cond_ld, bool forward);
  void launch_attn(const float* qkv, float* ao, const EncLayerW& L, int Hc, const int* lens, const int* offs, int maxLen, Planes* pl);
  void bind_weights();
  void bind_flow_decoder();
  void bind_wn_encoder(const std::string& p, int cin);
  void launch_conv(const std::vector<ConvP>& ps, int rmul, const int* lens, const int* offs, int maxLen, int nB);
  void encoder_layer(const EncLayerW& L, float*& x, float*& xb, float* qkv, float* ao, float* y, float* ffh, int Hc, int Fc,
                     int ks, const int* lens, const int* offs, int maxLen, const float* vec_after, int vec_ld,
                     const float* cadd_after);
  void dds_stack(const DdsW* d, int C, int k, float*& a, float*& b, const int* lens, const int* offs, int maxLen,
                 const float* x0 = nullptr, const float* pre_w = nullptr, const float* pre_b = nullptr, const float* cond = nullptr);
  struct P1Pin { int *len, *off, *sid, *ids; float *prm, *eps; };
  P1Pin p1_layout(int t_max, bool eps);
  void stage1(const int* ids_packed_host, const int* sid_host, int t_max, const float* noise_dp_host);
  void finish1();
  Planes enc_px;                               // the text encoder's output planes (precision modes 2 / 3), read by prior_stats
  void text_encoder(const float* cond, int cond_ld);
  void prior_stats();
  void phase1(const int* ids_packed_host, const int64_t* d_ids64, int t_max, const int64_t* d_sid64, const int* sid_host,
              const float* noise_dp, bool noise_on_device);
  void phase2(const float* noise_z, int z_ld, bool noise_on_device, bool run_decoder = true);
  void stage_noise_z(const float* noise_z, int z_ld) {       // caller memory (maybe pageable) -> pinned [B][I][maxFrm]
    const int I = cfg.inter_channels;
    float* pin = reinterpret_cast<float*>(ensure_pinned(h_pin_z, (size_t)B * I * maxFrm * sizeof(float)));
    const size_t ncopy = (size_t)std::min(z_ld, maxFrm);
    for (long r = 0; r < (long)B * I; ++r) memcpy(pin + r * maxFrm, noise_z + r * (long)z_ld, ncopy * sizeof(float));
  }
  void decode(float* z, const int* fl, const int* fo, bool planes_ready = false, bool pz_ready = false);
  bool have_latent = false;
  Buf<int> d_chunk;                              // [len, off, off_end] of the chunk being decoded

  // WN stack (modules.py:148-176) shared by the flow's coupling layers and the posterior encoder: `x` (and, on the tensor
  // cores, its planes px) is updated in place, `skip` receives the summed skip halves (planes pskip from the last layer);
  // layer i adds the cond rows cond + i*2H (row stride cond_ld) before the gate, none when cond is null.
  void wn_ffma(const std::vector<ConvW>& in, const std::vector<ConvW>& rsx, const std::vector<ConvW>& rss, int nl, int fk,
               int dil_rate, float* x, float* acts, float* skip, const float* cond, int cond_ld, const int* fl, const int* fo);
  void wn_tc(const std::vector<TcW>& t_in, const std::vector<ConvW>& in, const std::vector<TcW>& t_rsx, const std::vector<ConvW>& rsx,
             const std::vector<TcW>& t_rss, const std::vector<ConvW>& rss, int nl, int fk, int dil_rate, float* x, float* skip, const Planes& px,
             const Planes& pacts, const Planes& pskip, const float* cond, int cond_ld, const int* fl, const int* fo);
  // The flow on the fp32 pipe; forward = models.py:750-753 (layers in order, x1 <- x1 + m), else the reverse of infer.
  void flow_ffma(float* z, const int* fl, const int* fo, const float* cond, int cond_ld, bool forward);

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
  Buf<float> d_vprm, d_vin, d_vlin, d_vfeat, d_vstats, d_vcsrc, d_vnoise, d_vz_dbg, d_vzp_dbg;
  Buf<char> h_pin_vc;
  struct VcPin { int *frm_len, *frm_off, *clip_len, *sid; float *prm, *in, *eps; };
  VcPin vc_layout(bool from_spec, bool eps);
  float* vc_upload(bool from_spec, bool eps);
  float* cond_src(bool tgt);
  float* front_end(bool from_spec);
  void posterior_encode(const float* feat, int feat_ld, const float* noise, const float* qcond, int qld);
  void posterior_side(bool from_spec, const float* noise, const float* csrc);
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
  Buf<float> d_units, d_qg;                        // content-unit rows [Tfrm][unit channels], g [B][gin]
  Buf<char> h_pin_qv;
  struct QvPin { int *frm_len, *frm_off, *ident; float *prm, *units, *g, *eps; };
  QvPin qv_layout(bool eps);
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
  Buf<char> h_pin_cv;
  void bind_contentvec();
  std::vector<int> cv_stage(const float* wav, const int64_t* lengths, int64_t ld);
  void cv_enqueue(float* out, const int* out_offs);

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
  REQUIRE(c.dp_num_bins <= SPL_MAXB, VTTS_ERR_INVALID, "too many spline bins");
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
  tc = c.precision >= 1 && c.precision <= 3;
  dec_pre = conv("dec.pre", I, c.upsample_initial_channel, 7, !tc);
  if (tc) {
    REQUIRE(c.decoder_type == 0 && c.resblock_type == 1, VTTS_ERR_INVALID, "tensor-core mode supports the MB-iSTFT / ResBlock1 decoder");
    tc_pre = tcw("dec.pre", I, c.upsample_initial_channel, 7);
  }
  ups.clear();
  rbs.clear();
  int ch = c.upsample_initial_channel;
  up_total = 1;
  for (int i = 0; i < c.n_upsamples; ++i) {
    // ConvTranspose1d padding: (K-u)/2 in VITS2 (training/vits2/models.py:857-858, 989-990), (K-u+1-i)/2 with output_padding 1-i in
    // QuickVC (vc/models.py:428-430); both make exactly u*T output rows (config.convt_pad checks QuickVC's)
    const int u = c.upsample_rates[i], K = c.upsample_kernel_sizes[i];
    const int p = c.model_family == VTTS_FAMILY_QUICKVC ? (K - u + 1 - i) / 2 : (K - u) / 2;
    UpW U;
    for (int r = 0; r < u; ++r) {
      // polyphase split of ConvTranspose1d (see weights.convt_phases): taps per phase and left padding
      int d_min = -((r + p) / u);
      int d_max = (K - 1 - r - p) / u;
      U.phase.push_back(conv("dec.up" + std::to_string(i) + ".p" + std::to_string(r), ch, ch / 2, d_max - d_min + 1, !tc));
      if (tc) U.tphase.push_back(tcw("dec.up" + std::to_string(i) + ".p" + std::to_string(r), ch, ch / 2, d_max - d_min + 1));
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
          R.c1.push_back(conv(p2 + ".c1." + std::to_string(d), ch, ch, c.resblock_kernel_sizes[j], !tc));
          R.c2.push_back(conv(p2 + ".c2." + std::to_string(d), ch, ch, c.resblock_kernel_sizes[j], !tc));
          if (tc) {
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
void vtts_engine::launch_tc(const std::vector<TcSpec>& ps, int rmul, const int* lens, const int* offs, int maxLen, int nB) {
  // 128-wide channel tiles halve the activation traffic and run the MMA at its smem-operand optimum, but halve the CTA
  // count: used once the launch still fills the machine (batched calls), or when forced (VTTS_TC_BN).
  int BN = 64;
  {
    const std::vector<int>& hl = (lens == d_tok_len.p) ? v_tok_len : v_frm_len;
    long ctas128 = 0;
    bool wide = true;
    for (const TcSpec& q : ps) {
      if (q.Cout < 128) wide = false;
      for (int b = 0; b < nB; ++b) ctas128 += (long)((hl[b] * rmul + q.in_extra + TC_BM - 1) / TC_BM) * ((q.Cout + 127) / 128);
    }
    if (wide && ctas128 >= 2 * n_sm) BN = 128;
    if (tc_bn == 64 || tc_bn == 128) BN = tc_bn;
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
  if (tc_tall <= 0 && tc_split != 1 && (tc_bn == 64 || tc_bn == 128 || BN == 64)) {
    const std::vector<int>& hl = (lens == d_tok_len.p) ? v_tok_len : v_frm_len;
    TcSplitIn in;
    in.n = (int)ps.size(); in.nb = nB; in.gx = gx;
    in.bn = (tc_bn == 64 || tc_bn == 128) ? tc_bn : 0;
    in.max_split = tc_split > 1 ? tc_split : 8;
    in.min_steps = tc_min_steps;
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
  const bool big = tc_persist == 2 || (tc_persist && grid_tiles > (long)tc_persist_min * n_sm);   // (2: forced, for tests)
  bool tall = split == 1 && (tc_tall > 0 || (tc_tall == 0 && big));
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
  if (tc_mc && !tall) {
    int ny = -1;
    bool same = true;
    for (const TcSpec& q : ps) {
      const int n = (q.Cout + BN - 1) / BN;
      if (ny < 0) ny = n; else if (n != ny) same = false;
    }
    if (same) cn = (ny % 4 == 0) ? 4 : (ny % 2 == 0 ? 2 : 1);
    if (tc_mc == 2 && same && ny % 2 == 0) cn = 2;          // VTTS_TC_MULTICAST=2: pairs only
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
  const bool one_wave = tiles_all <= n_sm && !(tc_persist == 2 && split == 1 && cn == 1);
  tb.wst = np == 3 ? (BN == 128 ? 2 : 3) : (BN == 128 ? tc_wst<128>() : tc_wst<64>());
  tb.split = split;
  tb.cn = cn;
  tb.tall = tall ? 1 : 0;
  // persistent launches: CTA pairs share every weight tile through TMA multicast (conv_tc.cuh)
  const int wmc = (big && tc_wmc && split == 1 && cn == 1 && np == 2 && n_sm % 2 == 0) ? 2 : 1;
  tb.baseoff = tc_baseoff;
  tb.dbgskip = tc_dbgskip;
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
  if (split == 1 && cn == 1 && !tb.wpre && (tc_persist == 2 || (tc_persist && (long)grid.x * grid.y * grid.z > (long)tc_persist_min * n_sm))) {
    tb.persist = 1;
    tb.wmc = wmc;
    grid = dim3((unsigned)n_sm, 1, 1);
  }
  REQUIRE(tb.persist || wmc == 1, VTTS_ERR_INVALID, "tensor-core conv: weight multicast planned for a launch that is not persistent");
  const bool single_wave_image = split > 1 || tb.wpre;
  const bool dyn_image = tb.np != 2 || tb.ast != (BN == 128 ? tc_ast<128>() : tc_ast<64>()) || tb.wst != (BN == 128 ? tc_wst<128>() : tc_wst<64>());
  {
    vtts_conv_report r{};
    r.use_tc = 1; r.bn = BN; r.split = split; r.tall = tb.tall; r.cn = cn; r.wmc = tb.wmc; r.persist = tb.persist; r.np = tb.np;
    r.ast = tb.ast; r.wst = tb.wst; r.image = single_wave_image ? (dyn_image ? 1 : 0) : 2;
    r.grid_x = (int)grid.x; r.grid_y = (int)grid.y; r.grid_z = (int)grid.z;
    for (size_t p = 0; p < ps.size(); ++p) r.psplit[p] = psplit[p];
    note_conv(r);
  }
  if (profiling) {
    if (tc_prof_used + 2 > tc_prof_ev.size()) {
      tc_prof_ev.resize(tc_prof_used + 2);
      CK(cudaEventCreate(&tc_prof_ev[tc_prof_used]));
      CK(cudaEventCreate(&tc_prof_ev[tc_prof_used + 1]));
    }
    for (const TcSpec& q : ps)
      for (int b = 0; b < nB; ++b)
        tc_prof_flops += 2.0 * ((double)((lens == d_tok_len.p) ? h_tok_len[b] : h_frm_len[b]) * rmul + q.in_extra) * q.Cout * q.Cin * q.k;   // (true lengths)
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
        if (BN == 128) CK(cudaLaunchKernelEx(&lc, conv_tc_kernel<128, true>, tb, lens, offs));
        else CK(cudaLaunchKernelEx(&lc, conv_tc_kernel<64, true>, tb, lens, offs));
      } else {                    // the default launches carry the descriptor without the third-plane tensor maps
        // (a one-slot descriptor for the single-conv launches was tried as well: alternating between two kernel images on the
        //  chain cost more than the 2 KB of parameters saved -- conv_tc 723 -> 765 us in-graph)
        const auto tl = tc_lite<TC_MAXP>(tb);
        if (BN == 128) CK(cudaLaunchKernelEx(&lc, conv_tc_kernel<128, false, TC_MAXP>, tl, lens, offs));
        else CK(cudaLaunchKernelEx(&lc, conv_tc_kernel<64, false, TC_MAXP>, tl, lens, offs));
      }
    } else {                      // more than one wave of tiles: the persistent kernel (also runs them one per CTA when tb.persist == 0)
      if (BN == 128) CK(cudaLaunchKernelEx(&lc, conv_tc_persist_kernel<128>, tb, lens, offs));
      else CK(cudaLaunchKernelEx(&lc, conv_tc_persist_kernel<64>, tb, lens, offs));
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
bool vtts_engine::attn_tc_ok(const EncLayerW& L, int Hc) const {
  const int dk = Hc / L.heads;
  return attn_tc_mode > 0 && L.rk_hi != nullptr && dk % 32 == 0 && dk <= 128 && 2 * cfg.window_size + 1 <= ATC_RS && (3 * Hc) % 8 == 0;
}
// Which attention kernel for this launch?  The tensor-core kernel wins as soon as the launch is throughput bound (batches,
// long utterances: 8.8x at 4765 frames, 2.8x on the flow of a 64-utterance batch).  A single short utterance is latency
// bound -- a 128-row wgmma tile walks its 2-4 key tiles serially while the split-KV FFMA kernel spreads 4 query rows x 4
// key segments over 16 warps of ~80 CTAs -- and keeps the FFMA kernel (measured at 162 frames: 6 vs 19 us per launch in the
// graph).  VTTS_ATTN_TC = 0 never / 1 this rule / 2 always.
bool vtts_engine::attn_use_tc(const EncLayerW& L, int Hc, const int* lens, int maxLen) const {
  if (!attn_tc_ok(L, Hc)) return false;
  if (attn_tc_mode >= 2) return true;
  return !((attn_rows == 0 || attn_rows == 1) && attn_split_fits(L, Hc, lens, maxLen));
}

// Can the split-KV FFMA kernel take this launch?  All key tiles of the longest utterance must be resident in shared memory
// (at most ATS_MAXT tiles, and at most ATS_SMEM_MAX bytes: dk 128 at W 4 overflows from 7 tiles, i.e. 193 positions), and
// the CTAs must fit one wave.
bool vtts_engine::attn_split_fits(const EncLayerW& L, int Hc, const int* lens, int maxLen) const {
  const int dk = Hc / L.heads, nrel = 2 * cfg.window_size + 1;
  const std::vector<int>& hl = (lens == d_tok_len.p) ? v_tok_len : v_frm_len;
  long ctas = 0;
  for (int b = 0; b < B; ++b) ctas += (long)((hl[b] + ATS_ROWS - 1) / ATS_ROWS) * L.heads;
  const int mt = (maxLen + AT_KT - 1) / AT_KT;
  return attn_split && mt <= ATS_MAXT && ctas <= n_sm && dk % 32 == 0 && dk <= 128 &&
         (long)attn_split_smem_floats(dk, nrel, mt) * (long)sizeof(float) <= ATS_SMEM_MAX;
}

void vtts_engine::launch_attn_tc(const Planes& qkv, float* ao, Planes* pl, const EncLayerW& L, int Hc, const int* lens, const int* offs, int maxLen) {
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
  dim3 grid((maxLen + ATC_BM - 1) / ATC_BM, L.heads, B);
  if (grid.x == 0) return;
  last_attn = vtts_attn_report{VTTS_ATTN_TC, dk, 0, (int)grid.x, (int)grid.y, (int)grid.z, atc_smem_bytes(dk)};
  switch (dk / 32) {
    case 1: klaunch(attn_tc_kernel<32>, grid, dim3(ATC_THREADS), (size_t)atc_smem_bytes(32), ap, lens, offs); break;
    case 2: klaunch(attn_tc_kernel<64>, grid, dim3(ATC_THREADS), (size_t)atc_smem_bytes(64), ap, lens, offs); break;
    case 3: klaunch(attn_tc_kernel<96>, grid, dim3(ATC_THREADS), (size_t)atc_smem_bytes(96), ap, lens, offs); break;
    default: klaunch(attn_tc_kernel<128>, grid, dim3(ATC_THREADS), (size_t)atc_smem_bytes(128), ap, lens, offs); break;
  }
  CK(cudaGetLastError());
  ++launches;
}

void vtts_engine::launch_attn(const float* qkv, float* ao, const EncLayerW& L, int Hc, const int* lens, const int* offs, int maxLen, Planes* pl) {
  const int n_heads = L.heads;
  const int dk = Hc / n_heads, nrel = 2 * cfg.window_size + 1;
  __nv_bfloat16* ph = pl ? pl->hi : nullptr;
  __nv_bfloat16* plo = pl ? pl->lo : nullptr;
  __nv_bfloat16* pmi = pl ? pl->mid : nullptr;
  // register-blocked variant (4 query rows per warp) once the launch is throughput bound
  const std::vector<int>& hl = (lens == d_tok_len.p) ? v_tok_len : v_frm_len;
  long rows = 0;
  for (int b = 0; b < B; ++b) rows += hl[b];
  const int R = (attn_rows == 1 || attn_rows == 4) ? attn_rows : (rows * n_heads >= 8L * 2 * n_sm * 4 ? 4 : 1);
  // single short utterances: split-KV variant (all K/V tiles resident, 4 warps per query row) when it fits one wave
  {
    const int mt = (maxLen + AT_KT - 1) / AT_KT;
    if (R == 1 && attn_split_fits(L, Hc, lens, maxLen)) {
      dim3 grid((maxLen + ATS_ROWS - 1) / ATS_ROWS, n_heads, B);
      const size_t smem = (size_t)attn_split_smem_floats(dk, nrel, mt) * sizeof(float);
      last_attn = vtts_attn_report{VTTS_ATTN_SPLIT, dk, 1, (int)grid.x, (int)grid.y, (int)grid.z, (int)smem};
#define ATTN_SPLIT(D) klaunch(attn_split_kernel<D>, grid, dim3(ATS_THREADS), smem, qkv, 3 * Hc, ao, Hc, L.relk, L.relv, n_heads, cfg.window_size, mt, lens, offs, ph, plo, pmi)
      switch (dk / 32) { case 1: ATTN_SPLIT(1); break; case 2: ATTN_SPLIT(2); break; case 3: ATTN_SPLIT(3); break; default: ATTN_SPLIT(4); break; }
#undef ATTN_SPLIT
      CK(cudaGetLastError());
      ++launches;
      return;
    }
  }
  const int QT = 8 * R;
  dim3 grid((maxLen + QT - 1) / QT, n_heads, B);
  const size_t smem = (size_t)attn_smem_floats(dk, nrel, R) * sizeof(float);
  last_attn = vtts_attn_report{R == 4 ? VTTS_ATTN_R4 : VTTS_ATTN_R1, dk, R, (int)grid.x, (int)grid.y, (int)grid.z, (int)smem};
#define ATTN_CASE(D, RR) klaunch(attn_kernel<D, RR>, grid, dim3(AT_THREADS), smem, qkv, 3 * Hc, ao, Hc, L.relk, L.relv, n_heads, cfg.window_size, lens, offs, ph, plo, pmi)
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
  const int nk = c.n_resblock_kernels;
  int slot = 0;
  dcp.pz = planes(slot++, F, 1, c.inter_channels);
  dcp.cur = planes(slot++, F, 1, c.upsample_initial_channel);
  dcp.px.resize(c.n_upsamples); dcp.nxt.resize(c.n_upsamples); dcp.pj.resize(c.n_upsamples); dcp.pt.resize(c.n_upsamples);
  int rmp = 1, chp = c.upsample_initial_channel;
  for (int i = 0; i < c.n_upsamples; ++i) {
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
void vtts_engine::flow_tc(float* z, const int* fl, const int* fo, bool emit_pz, const float* cond, int cond_ld, bool forward) {
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
  dim3 lg((maxFrm + 3) / 4, B);
  for (int s = 0; s < nf; ++s) {
    const int f = forward ? s : nf - 1 - s;
    const FlowW& W = flow[f];
    const bool flipped = ((nf - f) % 2) == 1;
    const int x0off = flipped ? half : 0, x1off = flipped ? 0 : half;
    {
      ConvP p = mk(W.pre, z, I, x0off, h, H, 0, 1, 0);
      Planes& dst = c.use_transformer_flows ? ph : pwx;
      p.p_hi = dst.hi; p.p_lo = dst.lo; p.ldp = H; p.pl_slope = 1.f;
      launch_conv({p}, 1, fl, fo, maxFrm, B);
    }
    float* wn_x = h;
    if (c.use_transformer_flows) {
      if (attn_use_tc(W.tr, H, fl, maxFrm)) {
        // q, k, v leave the qkv conv as split-bf16 planes only; attention runs on wgmma (attn_tc.cuh)
        { TcSpec q; q.in = ph; q.w = W.t_qkv; q.bias = W.tr.qkv.b; q.Cin = H; q.Cout = 3 * H; q.out = pqkv; q.pl_slope = 1.f;
          launch_tc({q}, 1, fl, fo, maxFrm, B); }
        launch_attn_tc(pqkv, nullptr, &pao, W.tr, H, fl, fo, maxFrm);
      } else {
        { TcSpec q; q.in = ph; q.w = W.t_qkv; q.bias = W.tr.qkv.b; q.Cin = H; q.Cout = 3 * H; q.y = fqkv; q.ldy = 3 * H;
          launch_tc({q}, 1, fl, fo, maxFrm, B); }
        launch_attn(fqkv, fao, W.tr, H, fl, fo, maxFrm, &pao);
      }
      { TcSpec q; q.in = pao; q.w = W.t_o; q.bias = W.tr.o.b; q.Cin = H; q.Cout = H; q.y = fy; q.ldy = H;
        launch_tc({q}, 1, fl, fo, maxFrm, B); }
      klaunch(add_ln_kernel, dim3(lg), dim3(128), (size_t)(0), h, fy, W.tr.ln1.g, W.tr.ln1.b, nullptr, nullptr, 0, h1, fl, fo, H, ph1.hi, ph1.lo, (__nv_bfloat16*)nullptr);
      CK(cudaGetLastError());
      ++launches;
      { TcSpec q; q.in = ph1; q.w = W.t_ffn1; q.bias = W.tr.ffn1.b; q.Cin = H; q.Cout = H; q.k = fk; q.pad = (fk - 1) / 2;
        q.epi = TCE_RELU; q.out = pff; q.pl_slope = 1.f;
        launch_tc({q}, 1, fl, fo, maxFrm, B); }
      { TcSpec q; q.in = pff; q.w = W.t_ffn2; q.bias = W.tr.ffn2.b; q.Cin = H; q.Cout = H; q.k = fk; q.pad = (fk - 1) / 2;
        q.y = fy; q.ldy = H;
        launch_tc({q}, 1, fl, fo, maxFrm, B); }
      klaunch(add_ln_kernel, dim3(lg), dim3(128), (size_t)(0), h1, fy, W.tr.ln2.g, W.tr.ln2.b, h, nullptr, 0, wx, fl, fo, H, pwx.hi, pwx.lo, (__nv_bfloat16*)nullptr);
      CK(cudaGetLastError());
      ++launches;
      wn_x = wx;
    }
    wn_tc(W.t_in, W.in, W.t_rsx, W.rsx, W.t_rss, W.rss, nl, fk, c.flow_dilation_rate, wn_x, skip, pwx, pacts, pskip,
          cond ? cond + r_flow + f * nl * 2 * H : nullptr, cond_ld, fl, fo);
    { TcSpec q; q.in = pskip; q.w = W.t_post; q.bias = W.post.b; q.Cin = H; q.Cout = half; q.alpha = forward ? 1.f : -1.f;
      q.y = z; q.ldy = I; q.yoff = x1off; q.res = z; q.ldr = I; q.roff = x1off;
      if (emit_pz && f <= 1) { q.out = dcp.pz; q.poff = x1off; q.pl_slope = 1.f; }     // this half of z is final now
      launch_tc({q}, 1, fl, fo, maxFrm, B); }
  }
}

void vtts_engine::wn_tc(const std::vector<TcW>& t_in, const std::vector<ConvW>& in, const std::vector<TcW>& t_rsx,
                        const std::vector<ConvW>& rsx, const std::vector<TcW>& t_rss, const std::vector<ConvW>& rss, int nl, int fk,
                        int dil_rate, float* x, float* skip, const Planes& px, const Planes& pacts, const Planes& pskip, const float* cond,
                        int cond_ld, const int* fl, const int* fo) {
  const int H = cfg.hidden_channels;
  int dil = 1;
  for (int i = 0; i < nl; ++i) {
    { TcSpec q; q.in = px; q.w = t_in[i]; q.bias = in[i].b; q.Cin = H; q.Cout = 2 * H; q.k = fk; q.dil = dil;
      q.pad = dil * (fk - 1) / 2; q.epi = TCE_GATE; q.out = pacts; q.pl_slope = 1.f;
      if (cond) { q.cond = cond + i * 2 * H; q.cond_ld = cond_ld; }
      launch_tc({q}, 1, fl, fo, maxFrm, B); }
    TcSpec qs; qs.in = pacts; qs.w = t_rss[i]; qs.bias = rss[i].b; qs.Cin = H; qs.Cout = H; qs.y = skip; qs.ldy = H;
    if (i > 0) { qs.res = skip; qs.ldr = H; }
    if (i < nl - 1) {
      TcSpec qx; qx.in = pacts; qx.w = t_rsx[i]; qx.bias = rsx[i].b; qx.Cin = H; qx.Cout = H; qx.y = x; qx.ldy = H;
      qx.res = x; qx.ldr = H; qx.out = px; qx.pl_slope = 1.f;
      launch_tc({qx, qs}, 1, fl, fo, maxFrm, B);
    } else {
      qs.out = pskip; qs.pl_slope = 1.f;
      launch_tc({qs}, 1, fl, fo, maxFrm, B);
    }
    dil *= dil_rate;
  }
}

// Decoder on the tensor cores (models.py:1016-1040): every conv consumes the split-bf16 planes written by its
// producer's epilogue; fp32 copies exist only where a residual or the MRF mean needs them.
void vtts_engine::decoder_tc(float* z, const int* fl, const int* fo, bool pz_ready) {
  const vtts_config& c = cfg;
  const int I = c.inter_channels;
  const long F = Tfrm;
  const int nk = c.n_resblock_kernels, nd = c.n_resblock_dilations;
  Planes pz = dcp.pz, cur = dcp.cur;
  const std::vector<Planes>&st_px = dcp.px, &st_nxt = dcp.nxt;
  const std::vector<std::vector<Planes>>&st_pj = dcp.pj, &st_pt = dcp.pt;
  if (!pz_ready) {
    dim3 g((maxFrm + EW_ROWS - 1) / EW_ROWS, B);
    klaunch(split_planes_kernel, dim3(g), dim3(EW_THREADS), (size_t)(0), z, I, pz.hi, pz.lo, I, I, 1.f, 0, 1, fl, fo);
    CK(cudaGetLastError());
    ++launches;
  }
  int ch = c.upsample_initial_channel;
  {
    TcSpec q;
    q.in = pz; q.w = tc_pre; q.bias = dec_pre.b; q.Cin = I; q.Cout = ch; q.k = 7; q.dil = 1; q.pad = 3;
    q.out = cur; q.pl_slope = 0.1f;
    if (r_dec >= 0) { q.cond = d_condv.p + r_dec; q.cond_ld = condR; }     // x = conv_pre(z) + cond(g) (QuickVC, vc/models.py:465)
    if (debug_flags & 1) { q.y = ensure(d_d0, (size_t)F * ch); q.ldy = ch; }
    launch_tc({q}, 1, fl, fo, maxFrm, B);
  }
  int rm = 1;
  if ((int)d_stage.size() < c.n_upsamples) {
    d_stage.resize(c.n_upsamples);
    d_xj.resize(c.n_upsamples);
    d_tmp.resize(c.n_upsamples);
    for (int i = 0; i < c.n_upsamples; ++i) { d_xj[i].resize(nk); d_tmp[i].resize(nk); }
  }
  float* lastX = nullptr;
  for (int i = 0; i < c.n_upsamples; ++i) {
    const int u = c.upsample_rates[i], ch2 = ch / 2;
    const long rows = F * rm * u;
    float* X = ensure(d_stage[i], (size_t)rows * ch2);
    Planes px = st_px[i];
    for (int r0 = 0; r0 < u; r0 += TC_MAXP) {
      std::vector<TcSpec> ps;
      for (int r = r0; r < std::min(u, r0 + TC_MAXP); ++r) {
        TcSpec q;
        q.in = cur; q.w = ups[i].tphase[r]; q.bias = ups[i].phase[r].b; q.Cin = ch; q.Cout = ch2;
        q.k = ups[i].phase[r].k; q.dil = 1; q.pad = ups[i].pad[r];
        q.y = X; q.ldy = ch2; q.out = px; q.pl_slope = 0.1f; q.out_mul = u; q.out_add = r;
        ps.push_back(q);
      }
      launch_tc(ps, rm, fl, fo, maxFrm, B);
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
    for (int b = 0; b < B; ++b) group_tiles += (long)nk * ((v_frm_len[b] * rm + TC_BM - 1) / TC_BM) * ((ch + 63) / 64);
    const bool branch = mrf_branch && !profiling && nk > 1 && nk - 1 <= 3 && group_tiles <= n_sm;
    if (branch) {
      struct Restore { cudaStream_t& s; cudaStream_t v; ~Restore() { s = v; } } restore{stream, stream};
      cudaStream_t main_stream = stream;
      CK(cudaEventRecord(ev_fork, main_stream));
      for (int j = nk - 1; j >= 0; --j) {              // largest kernel size first
        if (j > 0) {
          CK(cudaStreamWaitEvent(side[j - 1], ev_fork, 0));
          stream = side[j - 1];
        } else {
          stream = main_stream;
        }
        for (int d = 0; d < nd; ++d) {
          TcSpec a, b2;
          rb_pair(j, d, a, b2);
          launch_tc({a}, rm, fl, fo, maxFrm, B);
          launch_tc({b2}, rm, fl, fo, maxFrm, B);
        }
        if (j > 0) CK(cudaEventRecord(ev_join[j - 1], stream));
      }
      stream = main_stream;
      for (int j = 1; j < nk; ++j) CK(cudaStreamWaitEvent(main_stream, ev_join[j - 1], 0));
    } else {
      for (int d = 0; d < nd; ++d) {
        std::vector<TcSpec> p1(nk), p2(nk);
        // Launches of more than one wave (long utterances, batches) walk the tiles in problem order: the resblock with the
        // longest k-loop (largest kernel size) goes first, so that the last tiles are short ones.  Single-wave launches give
        // each resblock its own split instead (tc_split_plan), where the order does not matter.
        for (int j = 0; j < nk; ++j) rb_pair(j, d, p1[mrf_heavy_first ? nk - 1 - j : j], p2[mrf_heavy_first ? nk - 1 - j : j]);
        launch_tc(p1, rm, fl, fo, maxFrm, B);
        launch_tc(p2, rm, fl, fo, maxFrm, B);
      }
    }
    const bool last = (i + 1 == c.n_upsamples);
    Planes nxt = st_nxt[i];
    {
      dim3 g((maxFrm * rm + (last ? 1 : 0) + EW_ROWS - 1) / EW_ROWS, B);
      klaunch(mrf_mean_planes_kernel, dim3(g), dim3(EW_THREADS), (size_t)(0), xj[0], nk > 1 ? xj[1] : nullptr, nk > 2 ? xj[2] : nullptr, std::min(nk, 3),
                                                   (debug_flags & 1) ? X : nullptr, nxt.hi, nxt.lo, ch, last ? 0.01f : 0.1f,
                                                   last ? 1 : 0, rm, fl, fo);
      CK(cudaGetLastError());
      ++launches;
    }
    cur = nxt;
    lastX = X;
  }
  (void)lastX;
  const int cps = c.istft_n_fft + 2, pc = c.subbands * cps;
  float* post = ensure(d_post, ((size_t)F * rm + B) * pc);
  {
    TcSpec q;
    q.in = cur; q.w = tc_post; q.bias = dec_post.b; q.Cin = ch; q.Cout = pc; q.k = 7; q.dil = 1; q.pad = 3;
    q.y = post; q.ldy = pc; q.in_extra = 1; q.out_seq_extra = 1;
    launch_tc({q}, rm, fl, fo, maxFrm, B);
  }
  float* wav = ensure(d_wav, (size_t)F * hop + 16);
  const int M = maxFrm * rm * c.istft_hop;
  dim3 g((M + TL_M - 1) / TL_M, B);
  const size_t smem = ((size_t)tl_rec_frames(63, c.subbands, c.istft_n_fft, c.istft_hop) * pc + (size_t)c.subbands * (TL_M + 2 * tl_halo(63, c.subbands))) * sizeof(float);
  REQUIRE(c.istft_hop == 4 && c.istft_n_fft == 16, VTTS_ERR_INVALID, "iSTFT tail kernel is sized for n_fft=16, hop=4");
  klaunch(istft_pqmf_kernel, dim3(g), dim3(TL_THREADS), (size_t)(smem), post, pc, istft_basis, pqmf, c.subbands, c.istft_n_fft, c.istft_hop, 63, rm, fl, fo, wav, 0, 1, istft_w2);
  CK(cudaGetLastError());
  ++launches;
}

void vtts_engine::launch_conv(const std::vector<ConvP>& ps, int rmul, const int* lens, const int* offs, int maxLen, int nB) {
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
  const std::vector<int>& hl0 = (lens == d_tok_len.p) ? v_tok_len : v_frm_len;
  const std::vector<int>& hl_true = (lens == d_tok_len.p) ? h_tok_len : h_frm_len;
  long base0 = 0;
  for (const ConvP& q : ps)
    for (int b = 0; b < nB; ++b) base0 += (long)((hl0[b] * rmul + q.in_extra + CV_TT - 1) / CV_TT) * ((q.Cout + CV_TC - 1) / CV_TC);
  // many tiles (batched calls): one thread group per CTA (several CTAs per SM; r2, batch 64: 6.98 ms per step against 8.01 / 8.21
  // with 2 / 4 groups), no cluster.  Few tiles (batch 1): the k-steps of a tile are
  // spread over a cluster of S CTAs until the launch fills ~1 wave of SMs; ranks that still have long k-loops then get
  // 2-4 thread groups each (a lone warp per scheduler issues an FFMA only every other cycle).
  int G = base0 >= 2 * n_sm ? conv_big_g : conv_min_g;
  for (const ConvP& q : ps)
    while (G > 1 && q.Cin % (CV_CK * G) != 0) G >>= 1;
  auto min_steps = [&](int g) {
    int ms = 1 << 30;
    for (const ConvP& q : ps) ms = (q.Cin % (CV_CK * g) != 0) ? 0 : std::min(ms, q.Cin / (CV_CK * g) * q.k);
    return ms;
  };
  int S = 1;
  while (S < conv_max_s && base0 * S < conv_target && S * 2 <= min_steps(G)) S *= 2;
  const int xw = (CV_TT + maxHalo + 7) / 8 * 8 + 1;
  auto smem_floats = [&](int g) {
    const size_t pipe = (size_t)2 * CV_CK * g * xw + (size_t)CV_NS * CV_CK * g * CV_TC;
    return (std::max(pipe, (size_t)(g - 1) * 32 * CV_THREADS) + 3) / 4 * 4 + (size_t)32 * CV_THREADS;
  };
  if (conv_auto_g && base0 < 2 * n_sm)
    while (G * 2 <= conv_max_g && min_steps(G * 2) / S >= conv_auto_g && smem_floats(G * 2) * sizeof(float) <= (size_t)CONV_SMEM_MAX) G *= 2;
  REQUIRE(smem_floats(G) * sizeof(float) <= (size_t)CONV_SMEM_MAX, VTTS_ERR_INVALID, "conv tile does not fit in shared memory");
  cb.S = S;
  cb.xw = xw;
  const size_t pipe_floats = (size_t)2 * CV_CK * G * xw + (size_t)CV_NS * CV_CK * G * CV_TC;
  const size_t red_floats = (size_t)(G - 1) * 32 * CV_THREADS;
  const size_t stage_off = (std::max(pipe_floats, red_floats) + 3) / 4 * 4;
  cb.stage_off = (int)stage_off;
  const size_t smem = (stage_off + (S > 1 ? (size_t)32 * CV_THREADS : 0)) * sizeof(float);
  const std::vector<int>& hl = hl_true;      // (profiling FLOP count below)
  dim3 grid(((maxL + CV_TT - 1) / CV_TT) * S, (maxCout + CV_TC - 1) / CV_TC, nB * cb.n);
  if (grid.x == 0) return;
  {
    vtts_conv_report r{};
    r.S = S; r.G = G;
    r.grid_x = (int)grid.x; r.grid_y = (int)grid.y; r.grid_z = (int)grid.z;
    note_conv(r);
  }
  if (profiling) {
    if (prof_used + 2 > prof_ev.size()) {
      prof_ev.resize(prof_used + 2);
      CK(cudaEventCreate(&prof_ev[prof_used]));
      CK(cudaEventCreate(&prof_ev[prof_used + 1]));
    }
    for (const ConvP& q : ps)
      for (int b = 0; b < nB; ++b)
        prof_flops += 2.0 * ((double)hl[b] * rmul + q.in_extra) * q.Cout * q.Cin * q.k;
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
      case 4: CK(cudaLaunchKernelEx(&lc, conv_kernel<4>, cb, lens, offs)); break;
      case 2: CK(cudaLaunchKernelEx(&lc, conv_kernel<2>, cb, lens, offs)); break;
      default: CK(cudaLaunchKernelEx(&lc, conv_kernel<1>, cb, lens, offs)); break;
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
                                int Fc, int ks, const int* lens, const int* offs, int maxLen, const float* vec_after, int vec_ld,
                                const float* cadd_after) {
  const int nB = B;
  launch_conv({mk(L.qkv, x, Hc, 0, qkv, 3 * Hc, 0, 1, 0)}, 1, lens, offs, maxLen, nB);
  launch_attn(qkv, ao, L, Hc, lens, offs, maxLen, nullptr);
  launch_conv({mk(L.o, ao, Hc, 0, y, Hc, 0, 1, 0)}, 1, lens, offs, maxLen, nB);
  dim3 lg((maxLen + 3) / 4, nB);
  klaunch(add_ln_kernel, dim3(lg), dim3(128), (size_t)(0), x, y, L.ln1.g, L.ln1.b, nullptr, nullptr, 0, xb, lens, offs, Hc, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr);
  CK(cudaGetLastError());
  ++launches;
  {
    ConvP p = mk(L.ffn1, xb, Hc, 0, ffh, Fc, 0, 1, (ks - 1) / 2);
    p.epi = EPI_RELU;
    launch_conv({p}, 1, lens, offs, maxLen, nB);
  }
  launch_conv({mk(L.ffn2, ffh, Fc, 0, y, Hc, 0, 1, (ks - 1) / 2)}, 1, lens, offs, maxLen, nB);
  klaunch(add_ln_kernel, dim3(lg), dim3(128), (size_t)(0), xb, y, L.ln2.g, L.ln2.b, cadd_after, vec_after, vec_ld, x, lens, offs, Hc, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr);
  CK(cudaGetLastError());
  ++launches;
}

void vtts_engine::dds_stack(const DdsW* d, int C, int k, float*& a, float*& b, const int* lens, const int* offs, int maxLen,
                            const float* x0, const float* pre_w, const float* pre_b, const float* cond) {
  int dil = 1;
  for (int i = 0; i < 3; ++i) {
    DdsP P;
    P.x = a; P.y = b;
    P.x0 = (i == 0) ? x0 : nullptr; P.pre_w = pre_w; P.pre_b = pre_b; P.cond = cond;
    P.sep_w = d[i].sep_w; P.sep_b = d[i].sep_b;
    P.ln1g = d[i].ln1.g; P.ln1b = d[i].ln1.b;
    P.pw_w = d[i].pw.w; P.pw_b = d[i].pw.b; P.ldw = d[i].pw.ldw;
    P.ln2g = d[i].ln2.g; P.ln2b = d[i].ln2.b;
    P.C = C; P.k = k; P.dil = dil;
    // (16 positions per CTA were tried for batched calls -- 4x less weight streaming per position -- and measured slower:
    //  duration stage 3.20 vs 2.95 ms at batch 64)
    dim3 grid((maxLen + DDS_TT - 1) / DDS_TT, B);
    const size_t smem = ((size_t)DDS_NS * DDS_CH * C + (size_t)C * DDS_TT + 8 * DDS_TT) * sizeof(float);
    klaunch(dds_layer_kernel<DDS_TT>, dim3(grid), dim3(C), (size_t)(smem), P, lens, offs);
    CK(cudaGetLastError());
    ++launches;
    std::swap(a, b);
    dil *= k;
  }
}

// ---------------------------------------------------------------------------------------------------
// Phase 1: speaker vector, TextEncoder, StochasticDurationPredictor(reverse), durations.
// ---------------------------------------------------------------------------------------------------
void vtts_engine::phase1(const int* ids_packed_host, const int64_t* d_ids64, int t_max, const int64_t* d_sid64,
                         const int* sid_host, const float* noise_dp, bool noise_on_device) {
  const vtts_config& c = cfg;
  const int H = c.hidden_channels, D = c.dp_filter_channels;
  const size_t T = (size_t)Ttok;
  if (!capturing) CK(cudaEventRecord(ev[0], stream));
  // ---- inputs (host data was staged into h_pin_in by stage1(); only device work is enqueued here)
  int* tl = ensure(d_tok_len, B);
  int* to = ensure(d_tok_off, B + 1);
  int* ids = ensure(d_ids, T);
  int* sid = ensure(d_sid, B);
  float* prm = ensure(d_prm, 8);
  {
    P1Pin pp = p1_layout(t_max, noise_dp && !noise_on_device);
    CK(cudaMemcpyAsync(tl, pp.len, B * sizeof(int), cudaMemcpyHostToDevice, stream));
    CK(cudaMemcpyAsync(to, pp.off, (B + 1) * sizeof(int), cudaMemcpyHostToDevice, stream));
    CK(cudaMemcpyAsync(prm, pp.prm, 8 * sizeof(float), cudaMemcpyHostToDevice, stream));
    if (ids_packed_host) {
      CK(cudaMemcpyAsync(ids, pp.ids, T * sizeof(int), cudaMemcpyHostToDevice, stream));
      CK(cudaMemcpyAsync(sid, pp.sid, B * sizeof(int), cudaMemcpyHostToDevice, stream));
    } else {
      dim3 g((maxTok + 127) / 128, B);
      klaunch(pack_ids_kernel, dim3(g), dim3(128), (size_t)(0), d_ids64, t_max, ids, tl, to);
      CK(cudaGetLastError());
      klaunch(cast_sid_kernel, dim3((B + 127) / 128), dim3(128), (size_t)(0), d_sid64, sid, B);
      CK(cudaGetLastError());
      launches += 2;
    }
    if (noise_dp && !noise_on_device) {      // staged as [B][2][maxTok] (stage1)
      float* de = ensure(d_eps_dp, (size_t)B * 2 * maxTok);
      CK(cudaMemcpyAsync(de, pp.eps, (size_t)B * 2 * maxTok * sizeof(float), cudaMemcpyHostToDevice, stream));
      noise_dp = de;
    }
  }
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
  float* h29 = ensure(d_h29, T * 32);
  float* za = ensure(d_za, T);
  float* zb = ensure(d_zb, T);
  {
    ConvP p = mk(dp_pre, x, H, 0, dA, D, 0, 1, 0);
    if (has_g) { p.cond = condv + r_dp; p.cond_ld = condR; }
    launch_conv({p}, 1, tl, to, maxTok, B);
  }
  {
    float *a = dA, *b = dB;
    dds_stack(dp_dds, D, c.dp_kernel_size, a, b, tl, to, maxTok);
    launch_conv({mk(dp_proj, a, D, 0, dx, D, 0, 1, 0)}, 1, tl, to, maxTok, B);
  }
  {
    dim3 g((maxTok + 127) / 128, B);
    klaunch(dp_noise_kernel, dim3(g), dim3(128), (size_t)(0), noise_dp, eps_dp_ld, prm, za, zb, tl, to);
    CK(cudaGetLastError());
    ++launches;
  }
  float* cvar = zb;   // conditioning half (x0 after the Flip)
  float* tvar = za;   // transformed half (x1)
  const int nbins = c.dp_num_bins;
  REQUIRE(3 * nbins - 1 <= 32, VTTS_ERR_INVALID, "spline parameter row too wide");
  for (int n = c.dp_n_flows; n >= 2; --n) {
    const CfW& F = cf[n - 2];
    // (the ConvFlow front h = pre(x0) + cond, modules.py:366-367, is computed inside the first DDS layer)
    float *a = dA, *b = dB;
    dds_stack(F.dds, D, c.dp_kernel_size, a, b, tl, to, maxTok, cvar, F.pre_w, F.pre_b, dx);
    launch_conv({mk(F.proj, a, D, 0, h29, 32, 0, 1, 0)}, 1, tl, to, maxTok, B);
    {
      dim3 g((maxTok + 127) / 128, B);
      klaunch(spline_inverse_kernel, dim3(g), dim3(128), (size_t)(0), h29, 32, tvar, nbins, c.dp_tail_bound, sqrtf((float)D), tl, to);
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
          (volatile int*)(use_poll ? d_map : nullptr), dctr, fl_real);
  CK(cudaGetLastError());
  ++launches;
  if (!capturing) CK(cudaEventRecord(ev[3], stream));
  if (!use_poll) {
    int* p_len = reinterpret_cast<int*>(ensure_pinned(h_pin_len, (size_t)(2 * B + 2) * sizeof(int)));
    CK(cudaMemcpyAsync(p_len, fl, B * sizeof(int), cudaMemcpyDeviceToHost, stream));
    CK(cudaMemcpyAsync(p_len + B, fo, (B + 1) * sizeof(int), cudaMemcpyDeviceToHost, stream));
  }
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
      encoder_layer(enc[i], x, xb, qkv, ao, y, ffh, H, Fc, c.kernel_size, tl, to, maxTok, va, cond_ld, nullptr);
      continue;
    }
    // precision mode 2: same layer with the four convs on wgmma (attentions.py:57-63)
    const EncLayerW& L = enc[i];
    const int ks = c.kernel_size;
    dim3 lg((maxTok + 3) / 4, B);
    if (attn_use_tc(L, H, tl, maxTok)) {
      { TcSpec q; q.in = px; q.w = L.t_qkv; q.bias = L.qkv.b; q.Cin = H; q.Cout = 3 * H; q.out = pqkv; q.pl_slope = 1.f;
        launch_tc({q}, 1, tl, to, maxTok, B); }
      launch_attn_tc(pqkv, nullptr, &pao, L, H, tl, to, maxTok);
    } else {
      { TcSpec q; q.in = px; q.w = L.t_qkv; q.bias = L.qkv.b; q.Cin = H; q.Cout = 3 * H; q.y = qkv; q.ldy = 3 * H;
        launch_tc({q}, 1, tl, to, maxTok, B); }
      launch_attn(qkv, ao, L, H, tl, to, maxTok, &pao);
    }
    { TcSpec q; q.in = pao; q.w = L.t_o; q.bias = L.o.b; q.Cin = H; q.Cout = H; q.y = y; q.ldy = H;
      launch_tc({q}, 1, tl, to, maxTok, B); }
    klaunch(add_ln_kernel, lg, dim3(128), (size_t)0, x, y, L.ln1.g, L.ln1.b, (const float*)nullptr, (const float*)nullptr, 0, xb, tl, to, H, px1.hi, px1.lo, px1.mid);
    ++launches;
    { TcSpec q; q.in = px1; q.w = L.t_ffn1; q.bias = L.ffn1.b; q.Cin = H; q.Cout = Fc; q.k = ks; q.pad = (ks - 1) / 2;
      q.epi = TCE_RELU; q.out = pff; q.pl_slope = 1.f;
      launch_tc({q}, 1, tl, to, maxTok, B); }
    { TcSpec q; q.in = pff; q.w = L.t_ffn2; q.bias = L.ffn2.b; q.Cin = Fc; q.Cout = H; q.k = ks; q.pad = (ks - 1) / 2;
      q.y = y; q.ldy = H;
      launch_tc({q}, 1, tl, to, maxTok, B); }
    klaunch(add_ln_kernel, lg, dim3(128), (size_t)0, xb, y, L.ln2.g, L.ln2.b, (const float*)nullptr, va, cond_ld, x, tl, to, H, px.hi, px.lo, px.mid);
    ++launches;
  }
}

// Prior statistics m_p, logs_p (models.py:323-325): enc_p.proj of text_encoder's output -> d_stats [Ttok][2I].
void vtts_engine::prior_stats() {
  const int H = cfg.hidden_channels, I = cfg.inter_channels;
  const int* tl = d_tok_len.p;
  const int* to = d_tok_off.p;
  float* stats = ensure(d_stats, (size_t)Ttok * 2 * I);
  if (enc_on_tc) {
    TcSpec q; q.in = enc_px; q.w = tc_encproj; q.bias = enc_proj.b; q.Cin = H; q.Cout = 2 * I; q.y = stats; q.ldy = 2 * I;
    launch_tc({q}, 1, tl, to, maxTok, B);
  } else {
    launch_conv({mk(enc_proj, d_x.p, H, 0, stats, 2 * I, 0, 1, 0)}, 1, tl, to, maxTok, B);
  }
}

// Host side of phase 1: stage the call's inputs in pinned memory (fixed layout, so a captured graph can re-read it).
vtts_engine::P1Pin vtts_engine::p1_layout(int t_max, bool eps) {
  const size_t T = (size_t)Ttok;
  (void)t_max;
  const size_t bytes = (size_t)(3 * B + 1) * sizeof(int) + T * sizeof(int) + 8 * sizeof(float) +
                       (eps ? (size_t)B * 2 * maxTok * sizeof(float) : 0) + 64;
  char* pin = ensure_pinned(h_pin_in, bytes);
  P1Pin pp;
  pp.len = reinterpret_cast<int*>(pin);
  pp.off = pp.len + B;
  pp.sid = pp.off + B + 1;
  pp.ids = pp.sid + B;
  pp.prm = reinterpret_cast<float*>(pp.ids + T);
  pp.eps = pp.prm + 8;
  return pp;
}

void vtts_engine::stage1(const int* ids_packed_host, const int* sid_host, int t_max, const float* noise_dp_host) {
  P1Pin pp = p1_layout(t_max, noise_dp_host != nullptr);
  memcpy(pp.len, h_tok_len.data(), B * sizeof(int));
  memcpy(pp.off, h_tok_off.data(), (B + 1) * sizeof(int));
  if (ids_packed_host) {
    memcpy(pp.ids, ids_packed_host, (size_t)real_Ttok * sizeof(int));
    memcpy(pp.sid, sid_host, B * sizeof(int));
  }
  pp.prm[0] = scales[0]; pp.prm[1] = scales[1]; pp.prm[2] = scales[2]; pp.prm[3] = 0.f;
  const uint32_t lo = (uint32_t)seed, hi = (uint32_t)(seed >> 32);
  memcpy(&pp.prm[4], &lo, 4);
  memcpy(&pp.prm[5], &hi, 4);
  if (use_poll) {
    const size_t need = (size_t)(2 * B + 4);
    if (need > map_cap) {
      REQUIRE(!capturing, VTTS_ERR_STATE, "mapped buffer growth during capture");
      if (h_map) { CK(cudaStreamSynchronize(stream)); CK(cudaFreeHost(h_map)); h_map = nullptr; }
      map_cap = need + 256;
      CK(cudaHostAlloc(reinterpret_cast<void**>(&h_map), map_cap * sizeof(int), cudaHostAllocMapped));
      CK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&d_map), h_map, 0));
      h_map[0] = 0;
      ++ws_gen;
    }
    call_seq = (call_seq % 1000000) + 1;
    memcpy(&pp.prm[6], &call_seq, 4);
  } else {
    pp.prm[6] = 0.f;
  }
  memcpy(&pp.prm[7], &spec_cap, 4);        // frames the speculative second phase is sized for (0: none), see duration_kernel
  if (noise_dp_host) {        // [B][2][t_max] -> [B][2][maxTok]: the device layout depends on the length bucket only
    for (int r = 0; r < 2 * B; ++r)
      memcpy(pp.eps + (size_t)r * maxTok, noise_dp_host + (size_t)r * t_max, (size_t)std::min(t_max, maxTok) * sizeof(float));
    eps_dp_ld = maxTok;
  }
}

void vtts_engine::finish1() {
  if (use_poll) {
    // spin on the flag the last phase-1 kernel writes into mapped host memory (bounded; then fall back to a sync)
    volatile int* flag = h_map;
    bool seen = false;
    for (long spin = 0; spin < 40000000L; ++spin) {
      if (*flag == call_seq) { seen = true; break; }
      if ((spin & 0xFFFFF) == 0xFFFFF && cudaStreamQuery(stream) != cudaErrorNotReady) break;   // finished or failed
    }
    if (!seen) {
      CK(cudaStreamSynchronize(stream));
      REQUIRE(*flag == call_seq, VTTS_ERR_CUDA, "phase 1 finished without publishing the utterance lengths");
    }
    h_frm_len.assign(h_map + 1, h_map + 1 + B);
    h_frm_off.assign(h_map + 1 + B, h_map + 1 + 2 * B + 1);
    set_frame_shape();
    have_durations = true;
    return;
  }
  CK(cudaStreamSynchronize(stream));
  const int* p_len = reinterpret_cast<const int*>(h_pin_len.p);
  h_frm_len.assign(p_len, p_len + B);
  h_frm_off.assign(p_len + B, p_len + 2 * B + 1);
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
  if (!capturing) CK(cudaEventRecord(ev[4], stream));
  if (noise_z && !noise_on_device) {
    // host noise was staged into h_pin_z by the caller (stage_noise_z) as [B][I][maxFrm]: the layout depends on the bucket only
    const size_t n = (size_t)B * I * maxFrm;
    float* de = ensure(d_eps_z, n);
    CK(cudaMemcpyAsync(de, h_pin_z.p, n * sizeof(float), cudaMemcpyHostToDevice, stream));
    noise_z = de;
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
  if (flow_on_tc) flow_tc(z, fl, fo, emit_pz, cond, condR, /*forward=*/false);
  else flow_ffma(z, fl, fo, cond, condR, /*forward=*/false);
  if (!capturing) CK(cudaEventRecord(ev[5], stream));

  if (!run_decoder) return;
  decode(z, fl, fo, /*planes_ready=*/dec_now, /*pz_ready=*/emit_pz);
}

// Flow on the fp32 pipe (models.py:750-757).  Flip (modules.py:272-279) is folded into the packed pre/post weights: for a
// "flipped" layer x0 lives in physical channels [half, 2*half), x1 in [0, half).  forward / cond: see flow_tc.
void vtts_engine::flow_ffma(float* z, const int* fl, const int* fo, const float* cond, int cond_ld, bool forward) {
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
    launch_conv({mk(W.pre, z, I, x0off, h, H, 0, 1, 0)}, 1, fl, fo, maxFrm, B);
    float* wn_in = h;
    if (c.use_transformer_flows) {
      // h = h + Encoder(h)  (models.py:377): the layer's last LN adds `h` back and lands in wx
      float* xa = h; float* xb2 = h1;
      // encoder_layer writes its result into `xa` (== h) -- we need h preserved for the residual, so run the
      // layer on explicit buffers instead of the ping-pong helper:
      launch_conv({mk(W.tr.qkv, h, H, 0, fqkv, 3 * H, 0, 1, 0)}, 1, fl, fo, maxFrm, B);
      launch_attn(fqkv, fao, W.tr, H, fl, fo, maxFrm, nullptr);
      launch_conv({mk(W.tr.o, fao, H, 0, fy, H, 0, 1, 0)}, 1, fl, fo, maxFrm, B);
      dim3 lg((maxFrm + 3) / 4, B);
      klaunch(add_ln_kernel, dim3(lg), dim3(128), (size_t)(0), xa, fy, W.tr.ln1.g, W.tr.ln1.b, nullptr, nullptr, 0, xb2, fl, fo, H, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr);
      CK(cudaGetLastError());
      ++launches;
      {
        ConvP p = mk(W.tr.ffn1, xb2, H, 0, ffh2, H, 0, 1, (fk - 1) / 2);
        p.epi = EPI_RELU;
        launch_conv({p}, 1, fl, fo, maxFrm, B);
      }
      launch_conv({mk(W.tr.ffn2, ffh2, H, 0, fy, H, 0, 1, (fk - 1) / 2)}, 1, fl, fo, maxFrm, B);
      klaunch(add_ln_kernel, dim3(lg), dim3(128), (size_t)(0), xb2, fy, W.tr.ln2.g, W.tr.ln2.b, h, nullptr, 0, wx, fl, fo, H, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr);
      CK(cudaGetLastError());
      ++launches;
      wn_in = wx;
    }
    // WN (modules.py:148-176).  The hidden state is updated in place in `wn_in`.
    wn_ffma(W.in, W.rsx, W.rss, nl, fk, c.flow_dilation_rate, wn_in, acts, skip, cond ? cond + r_flow + f * nl * 2 * H : nullptr, cond_ld,
            fl, fo);
    {
      // x1 <- x1 - post(h) (reverse) / x1 + post(h) (forward) (mean_only; models.py:381-391)
      ConvP p = mk(W.post, skip, H, 0, z, I, x1off, 1, 0);
      p.alpha = forward ? 1.f : -1.f;
      p.res = z; p.ldr = I; p.roff = x1off;
      launch_conv({p}, 1, fl, fo, maxFrm, B);
    }
  }
}

void vtts_engine::wn_ffma(const std::vector<ConvW>& in, const std::vector<ConvW>& rsx, const std::vector<ConvW>& rss, int nl, int fk,
                          int dil_rate, float* x, float* acts, float* skip, const float* cond, int cond_ld, const int* fl, const int* fo) {
  const int H = cfg.hidden_channels;
  int dil = 1;
  for (int i = 0; i < nl; ++i) {
    {
      ConvP p = mk(in[i], x, H, 0, acts, H, 0, dil, dil * (fk - 1) / 2);
      p.epi = EPI_GATE;
      if (cond) { p.cond = cond + i * 2 * H; p.cond_ld = cond_ld; }
      launch_conv({p}, 1, fl, fo, maxFrm, B);
    }
    ConvP ps = mk(rss[i], acts, H, 0, skip, H, 0, 1, 0);
    if (i > 0) { ps.res = skip; ps.ldr = H; ps.roff = 0; }
    if (i < nl - 1) {
      ConvP px = mk(rsx[i], acts, H, 0, x, H, 0, 1, 0);
      px.res = x; px.ldr = H; px.roff = 0;
      launch_conv({px, ps}, 1, fl, fo, maxFrm, B);
    } else {
      launch_conv({ps}, 1, fl, fo, maxFrm, B);
    }
    dil *= dil_rate;
  }
}

// Decoder over the utterance rows described by (fl, fo) -- the whole batch, or one halo-extended chunk of a single
// utterance (vtts_decode_chunk).
void vtts_engine::decode(float* z, const int* fl, const int* fo, bool planes_ready, bool pz_ready) {
  const vtts_config& c = cfg;
  const int I = c.inter_channels;
  const size_t F = (size_t)Tfrm;
  // ---- decoder (models.py:1016-1054 / 872-891)
  if (tc) {
    if (!planes_ready) {          // (chunked decoding: the decoder runs on its own)
      begin_planes();
      alloc_decoder_planes();
      flush_tails(fl, fo);
    }
    decoder_tc(z, fl, fo, pz_ready);
    if (!capturing) CK(cudaEventRecord(ev[6], stream));
    return;
  }
  int ch = c.upsample_initial_channel;
  float* cur = ensure(d_d0, F * ch);
  {
    ConvP p = mk(dec_pre, z, I, 0, cur, ch, 0, 1, 3);
    if (r_dec >= 0) { p.cond = d_condv.p + r_dec; p.cond_ld = condR; }     // x = conv_pre(z) + cond(g)
    launch_conv({p}, 1, fl, fo, maxFrm, B);
  }
  int rm = 1;
  const int nk = c.n_resblock_kernels, nd = c.n_resblock_dilations;
  if ((int)d_stage.size() < c.n_upsamples) {
    d_stage.resize(c.n_upsamples);
    d_xj.resize(c.n_upsamples);
    d_tmp.resize(c.n_upsamples);
    for (int i = 0; i < c.n_upsamples; ++i) { d_xj[i].resize(nk); d_tmp[i].resize(nk); }
  }
  for (int i = 0; i < c.n_upsamples; ++i) {
    const int u = c.upsample_rates[i], ch2 = ch / 2;
    const size_t rows = F * rm * u;
    float* X = ensure(d_stage[i], rows * ch2);
    for (int r0 = 0; r0 < u; r0 += CV_MAXP) {
      std::vector<ConvP> ps;
      for (int r = r0; r < std::min(u, r0 + CV_MAXP); ++r) {
        ConvP p = mk(ups[i].phase[r], cur, ch, 0, X, ch2, 0, 1, ups[i].pad[r]);
        p.pro = PRO_LRELU; p.slope = 0.1f;
        p.out_mul = u; p.out_add = r;
        ps.push_back(p);
      }
      launch_conv(ps, rm, fl, fo, maxFrm, B);
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
      launch_conv(p1, rm, fl, fo, maxFrm, B);
      if (c.resblock_type == 1) {
        launch_conv(p2, rm, fl, fo, maxFrm, B);
      } else if (d > 0) {
        for (int j = 0; j < nk; ++j) std::swap(xj[j], tmp[j]);   // ResBlock2 ping-pong (halo reads forbid in-place)
      }
    }
    {
      REQUIRE(nk <= 3, VTTS_ERR_INVALID, "more than 3 resblocks per stage not supported");
      const long total4 = (long)(rows * ch / 4);
      klaunch(mrf_mean_kernel, dim3((unsigned)((total4 + 255) / 256)), dim3(256), (size_t)(0), xj[0], nk > 1 ? xj[1] : nullptr, nk > 2 ? xj[2] : nullptr,
                                                                           std::min(nk, 3), X, total4);
      CK(cudaGetLastError());
      ++launches;
    }
    cur = X;
  }
  float* wav = ensure(d_wav, F * hop + 16);
  if (c.decoder_type == 0) {
    const int cps = c.istft_n_fft + 2, pc = c.subbands * cps;
    float* post = ensure(d_post, (F * rm + B) * pc);
    ConvP p = mk(dec_post, cur, ch, 0, post, pc, 0, 1, 3);
    p.pro = PRO_LRELU; p.slope = 0.01f;
    p.reflect = 1; p.in_extra = 1; p.out_seq_extra = 1;
    launch_conv({p}, rm, fl, fo, maxFrm, B);
    const int M = maxFrm * rm * c.istft_hop;
    dim3 g((M + TL_M - 1) / TL_M, B);
    const size_t smem = ((size_t)tl_rec_frames(63, c.subbands, c.istft_n_fft, c.istft_hop) * pc + (size_t)c.subbands * (TL_M + 2 * tl_halo(63, c.subbands))) * sizeof(float);
    REQUIRE(c.istft_hop == 4 && c.istft_n_fft == 16, VTTS_ERR_INVALID, "iSTFT tail kernel is sized for n_fft=16, hop=4");
    klaunch(istft_pqmf_kernel, dim3(g), dim3(TL_THREADS), (size_t)(smem), post, pc, istft_basis, pqmf, c.subbands, c.istft_n_fft, c.istft_hop, 63, rm, fl, fo, wav, 0, 1, istft_w2);
    CK(cudaGetLastError());
    ++launches;
  } else {
    ConvP p = mk(dec_post, cur, ch, 0, wav, 1, 0, 1, 3);
    p.pro = PRO_LRELU; p.slope = 0.01f;
    p.epi = EPI_TANH;
    launch_conv({p}, rm, fl, fo, maxFrm, B);
  }
  if (!capturing) CK(cudaEventRecord(ev[6], stream));
}

// ---------------------------------------------------------------------------------------------------
// Voice conversion (models.py:1710-1718): spectrogram front end, enc_q with g_src, flow forward with g_src, flow reverse
// with g_tgt, decoder.  The frame counts follow from the input lengths, so the whole call is ONE graphed phase.
// ---------------------------------------------------------------------------------------------------
// Pinned staging of one call (fixed layout for a given batch / length bucket, so a captured graph re-reads it on replay):
// ints [frm_len B][frm_off B+1][clip_len B][sid_src B][sid_tgt B], prm[16], input (wav [B][vc_wld] or spec
// [B][spec_channels][maxFrm]), eps [B][inter][maxFrm].
vtts_engine::VcPin vtts_engine::vc_layout(bool from_spec, bool eps) {
  const vtts_config& c = cfg;
  const size_t nin = from_spec ? (size_t)B * c.spec_channels * maxFrm : (size_t)B * vc_wld;
  const size_t ints = (size_t)(5 * B + 1) * sizeof(int);
  const size_t head = (ints + 63) / 64 * 64;
  const size_t bytes = head + 16 * sizeof(float) + nin * sizeof(float) + (eps ? (size_t)B * c.inter_channels * maxFrm * sizeof(float) : 0) + 64;
  char* pin = ensure_pinned(h_pin_vc, bytes);
  VcPin pp;
  pp.frm_len = reinterpret_cast<int*>(pin);
  pp.frm_off = pp.frm_len + B;
  pp.clip_len = pp.frm_off + B + 1;
  pp.sid = pp.clip_len + B;
  pp.prm = reinterpret_cast<float*>(pin + head);
  pp.in = pp.prm + 16;
  pp.eps = pp.in + nin;
  return pp;
}

// Inputs of a call on the posterior side, from the pinned staging (vc_layout) to the device: frame lengths / offsets, clip
// lengths and speaker ids, the per-call scalars, the waveform or spectrogram, and the posterior eps (returned; null: Philox).
float* vtts_engine::vc_upload(bool from_spec, bool eps) {
  const vtts_config& c = cfg;
  const int I = c.inter_channels;
  VcPin pp = vc_layout(from_spec, eps);
  int* fl = ensure(d_frm_len, B);
  int* fo = ensure(d_frm_off, B + 1);
  int* vi = ensure(d_vint, 3 * B);                       // [clip_len B][sid_src B][sid_tgt B]
  float* prm = ensure(d_vprm, 16);
  const size_t nin = from_spec ? (size_t)B * c.spec_channels * maxFrm : (size_t)B * vc_wld;
  float* vin = ensure(d_vin, nin);
  CK(cudaMemcpyAsync(fl, pp.frm_len, B * sizeof(int), cudaMemcpyHostToDevice, stream));
  CK(cudaMemcpyAsync(fo, pp.frm_off, (B + 1) * sizeof(int), cudaMemcpyHostToDevice, stream));
  CK(cudaMemcpyAsync(vi, pp.clip_len, 3 * B * sizeof(int), cudaMemcpyHostToDevice, stream));
  CK(cudaMemcpyAsync(prm, pp.prm, 16 * sizeof(float), cudaMemcpyHostToDevice, stream));
  CK(cudaMemcpyAsync(vin, pp.in, nin * sizeof(float), cudaMemcpyHostToDevice, stream));
  float* noise = nullptr;
  if (eps) {
    noise = ensure(d_vnoise, (size_t)B * I * maxFrm);
    CK(cudaMemcpyAsync(noise, pp.eps, (size_t)B * I * maxFrm * sizeof(float), cudaMemcpyHostToDevice, stream));
  }
  return noise;
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
void vtts_engine::posterior_encode(const float* feat, int feat_ld, const float* noise, const float* qcond, int qld) {
  const vtts_config& c = cfg;
  const int H = c.hidden_channels, I = c.inter_channels;
  const size_t F = (size_t)Tfrm;
  const int* fl = d_frm_len.p;
  const int* fo = d_frm_off.p;
  float* h = ensure(d_h, F * H);
  float* acts = ensure(d_acts, F * H);
  float* skip = ensure(d_skip, F * H);
  float* stats = ensure(d_vstats, F * 2 * I);
  float* z = ensure(d_z, F * I);
  const bool flow_on_tc = tc && !flow.empty() && !flow[0].t_in.empty();
  if (flow_on_tc || q_tc) {
    begin_planes();
    alloc_flow_planes();                     // (enc_q uses the flow's WN planes before the flow runs)
    flush_tails(fl, fo);
  }
  {
    ConvP p = mk(q_pre, feat, feat_ld, 0, h, H, 0, 1, 0);
    if (q_tc) { p.p_hi = flp.pwx.hi; p.p_lo = flp.pwx.lo; p.ldp = H; p.pl_slope = 1.f; }
    launch_conv({p}, 1, fl, fo, maxFrm, B);
  }
  if (q_tc) {
    wn_tc(qt_in, q_in, qt_rsx, q_rsx, qt_rss, q_rss, Q_LAYERS, Q_KERNEL, 1, h, skip, flp.pwx, flp.pacts, flp.pskip, qcond, qld, fl, fo);
    TcSpec q; q.in = flp.pskip; q.w = qt_proj; q.bias = q_proj.b; q.Cin = H; q.Cout = 2 * I; q.y = stats; q.ldy = 2 * I;
    launch_tc({q}, 1, fl, fo, maxFrm, B);
  } else {
    wn_ffma(q_in, q_rsx, q_rss, Q_LAYERS, Q_KERNEL, 1, h, acts, skip, qcond, qld, fl, fo);
    launch_conv({mk(q_proj, skip, H, 0, stats, 2 * I, 0, 1, 0)}, 1, fl, fo, maxFrm, B);
  }
  klaunch(posterior_sample_kernel, dim3(maxFrm, B), dim3(64), (size_t)0, (const float*)stats, I, noise, maxFrm,
          (const float*)d_vprm.p, fl, fo, z);
  CK(cudaGetLastError());
  ++launches;
  if (debug_flags & 1) CK(cudaMemcpyAsync(ensure(d_vz_dbg, F * I), z, F * I * sizeof(float), cudaMemcpyDeviceToDevice, stream));
}

void vtts_engine::posterior_side(bool from_spec, const float* noise, const float* csrc) {
  const int I = cfg.inter_channels;
  const size_t F = (size_t)Tfrm;
  const int qld = condR + q_R;
  const int* fl = d_frm_len.p;
  const int* fo = d_frm_off.p;
  // ---- enc_q input rows [F][spec_pad]
  float* feat = front_end(from_spec);
  // ---- posterior encoder (models.py:836-842): pre -> 16-layer WN (g_src) -> proj -> sample
  posterior_encode(feat, spec_pad, noise, csrc ? csrc + condR : nullptr, qld);
  float* z = d_z.p;
  // ---- z_p = flow(z, g_src)   (models.py:1715, 1640)
  const bool flow_on_tc = tc && !flow.empty() && !flow[0].t_in.empty();
  if (flow_on_tc) flow_tc(z, fl, fo, false, csrc, qld, /*forward=*/true);
  else flow_ffma(z, fl, fo, csrc, qld, /*forward=*/true);
  if (debug_flags & 1) CK(cudaMemcpyAsync(ensure(d_vzp_dbg, F * I), z, F * I * sizeof(float), cudaMemcpyDeviceToDevice, stream));
}

void vtts_engine::convert_enqueue(bool from_spec, bool eps) {
  if (!capturing) CK(cudaEventRecord(ev[4], stream));
  const float* noise = vc_upload(from_spec, eps);
  // ---- g_src / g_tgt (models.py:1712-1713) and every cond row of both, one launch: src -> d_vcsrc [B][condR + q_R]
  //      (the TTS rows, then enc_q's), tgt -> d_condv [B][condR] (where the reverse flow and the decoder read them)
  const float* csrc = cond_src(/*tgt=*/true);
  const float* ctgt = d_condv.p;
  posterior_side(from_spec, noise, csrc);
  // ---- z_hat = flow^-1(z_p, g_tgt)   (models.py:1716)
  const int* fl = d_frm_len.p;
  const int* fo = d_frm_off.p;
  float* z = d_z.p;
  const bool flow_on_tc = tc && !flow.empty() && !flow[0].t_in.empty();
  if (flow_on_tc) flow_tc(z, fl, fo, false, ctgt, condR, /*forward=*/false);
  else flow_ffma(z, fl, fo, ctgt, condR, /*forward=*/false);
  if (!capturing) CK(cudaEventRecord(ev[5], stream));
  // ---- o_hat = dec(z_hat * y_mask, g=g_tgt)   (models.py:1717)
  decode(z, fl, fo);
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
  const float* noise = vc_upload(from_spec, eps);
  int* tl = ensure(d_tok_len, B);
  int* to = ensure(d_tok_off, B + 1);
  int* ids = ensure(d_ids, Ttok);
  {
    P1Pin pp = p1_layout(0, false);                    // (staged by the host: lengths, offsets, packed ids)
    CK(cudaMemcpyAsync(tl, pp.len, B * sizeof(int), cudaMemcpyHostToDevice, stream));
    CK(cudaMemcpyAsync(to, pp.off, (B + 1) * sizeof(int), cudaMemcpyHostToDevice, stream));
    CK(cudaMemcpyAsync(ids, pp.ids, (size_t)Ttok * sizeof(int), cudaMemcpyHostToDevice, stream));
  }
  const int* fl = d_frm_len.p;
  const int* fo = d_frm_off.p;
  const float* csrc = has_g ? cond_src(/*tgt=*/false) : nullptr;
  // ---- m_p, logs_p = enc_p(x, g)   (models.py:1632-1633)
  text_encoder(csrc, condR + q_R);
  prior_stats();
  if (!capturing) CK(cudaEventRecord(ev[2], stream));
  // ---- z_p = flow(enc_q(y, g), g)   (models.py:1639-1640)
  posterior_side(from_spec, noise, csrc);
  if (!capturing) CK(cudaEventRecord(ev[4], stream));
  // ---- neg_cent [B][T_y][T_x] over the frame and token buckets (models.py:1645-1651), then MAS (:1656-1660)
  const int Ty = maxFrm, Tx = maxTok;
  float* nc = ensure(d_ncent, (size_t)B * Ty * Tx);
  if (debug_flags & 1) CK(cudaMemsetAsync(nc, 0xFF, (size_t)B * Ty * Tx * sizeof(float), stream));   // NaN outside the utterances
  klaunch(neg_cent_kernel, dim3((Tx + NC_T - 1) / NC_T, (Ty + NC_T - 1) / NC_T, B), dim3(NC_THREADS), (size_t)0, (const float*)d_z.p,
          (const float*)d_stats.p, I, fl, fo, (const int*)tl, (const int*)to, nc, Ty, Tx);
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
  klaunch(mas_kernel, dim3(B), dim3(MAS_THREADS), (size_t)2 * Tx * sizeof(float), nc, (int*)nullptr, fl, (const int*)tl, Ty, Tx, tof, fo,
          dur, (const int*)to, score);
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
  const size_t head = ((size_t)cvp.nint * sizeof(int) + 63) / 64 * 64;
  const size_t nsamp = (size_t)cvp.tot0 * s0 + K0;
  char* pin = ensure_pinned(h_pin_cv, head + nsamp * sizeof(float) + 64);
  memcpy(pin, h.data(), (size_t)(2 * NL + 1) * B * sizeof(int));
  float* ps = reinterpret_cast<float*>(pin + head);
  for (int b = 0; b < B; ++b) {
    const int L0 = h[b];
    const int64_t need = std::min<int64_t>(lengths[b], (int64_t)(L0 - 1) * s0 + K0);
    const float* src = wav + (size_t)b * ld;
    memcpy(ps + h[2 * NL * B + b], src, (size_t)need * sizeof(float));
    double sum = 0.0;                                  // the clip's mean, in one fixed order (layer 0 runs centred on it)
    for (int64_t i = 0; i < lengths[b]; ++i) sum += src[i];
    const float mu = (float)(sum / (double)lengths[b]);
    memcpy(pin + ((2 * NL + 1) * B + b) * sizeof(int), &mu, sizeof(float));
  }
  return frames;
}

// ContentVec of the staged clips (cv_stage): layer 0 + GroupNorm + GELU, layers 1.. (conv_kernel over the strided row view,
// GELU epilogue), LayerNorm + projection, the grouped positional conv (two launches of half the taps each: the tile halo of
// conv_kernel), LayerNorm(x + gelu(pos)), then the post-LN transformer layers.  The last LayerNorm writes frame t of clip b
// to out row out_offs[b] + t (out_offs null: the frame level's own offsets).
void vtts_engine::cv_enqueue(float* out, const int* out_offs) {
  const vtts_config& c = cfg;
  const int NL = c.cv_n_conv, C = c.cv_conv_dim, H = c.cv_hidden, Fh = c.cv_ffn, K0 = c.cv_conv_kernel[0], s0 = c.cv_conv_stride[0];
  // The tensor-core GEMMs run without split-K (every output summed by one CTA in one k order, whatever its launch shape) and
  // attention on attn_tc_kernel whenever it takes the layer: a clip's units are then the same alone and in any batch.
  struct Saved {
    vtts_engine* e; std::vector<int> vf, hf; int split, atc;
    explicit Saved(vtts_engine* h) : e(h), vf(h->v_frm_len), hf(h->h_frm_len), split(h->tc_split), atc(h->attn_tc_mode) {}
    ~Saved() { e->v_frm_len = vf; e->h_frm_len = hf; e->tc_split = split; e->attn_tc_mode = atc; }
  } saved(this);
  if (cv_tc) {
    tc_split = 1;
    if (attn_tc_mode > 0) attn_tc_mode = 2;
  }
  const size_t head = ((size_t)cvp.nint * sizeof(int) + 63) / 64 * 64;
  const size_t nsamp = (size_t)cvp.tot0 * s0 + K0;
  int* di = ensure(d_cvi, cvp.nint);
  float* dw = ensure(d_cvwav, nsamp);
  CK(cudaMemcpyAsync(di, h_pin_cv.p, cvp.nint * sizeof(int), cudaMemcpyHostToDevice, stream));
  CK(cudaMemcpyAsync(dw, h_pin_cv.p + head, nsamp * sizeof(float), cudaMemcpyHostToDevice, stream));
  auto Ls = [&](int l) -> const int* { return di + l * B; };
  auto Os = [&](int l) -> const int* { return di + (NL + l) * B; };
  const int* woff = di + 2 * NL * B;
  const float* mu = reinterpret_cast<const float*>(di + (2 * NL + 1) * B);
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
  auto gelu = [&](float* y, int width, const int* lens, const int* offs, int maxLen, const Planes* pl) {
    klaunch(cv_gelu_kernel, dim3(maxLen, B), dim3(256), (size_t)0, y, width, lens, offs, pl ? pl->hi : (__nv_bfloat16*)nullptr,
            pl ? pl->lo : (__nv_bfloat16*)nullptr);
    CK(cudaGetLastError());
    ++launches;
  };
  float* x = lv[0];
  for (int i = 1; i < NL; ++i) {
    float* y = lv[i & 1];
    v_frm_len.assign(B, cvp.maxL[i]);
    h_frm_len = v_frm_len;
    launch_conv({mk(cv_conv[i], x, c.cv_conv_stride[i] * C, 0, y, C, 0, 1, 0)}, 1, Ls(i), Os(i), cvp.maxL[i], B);
    gelu(y, C, Ls(i), Os(i), cvp.maxL[i], nullptr);
    x = y;
  }
  const int* Lf = Ls(NL - 1);
  const int* Of = Os(NL - 1);
  const int maxF = cvp.maxL[NL - 1];
  const size_t Tf = (size_t)cvp.tot0 / cv_P;
  float *X = ensure(d_cvx, Tf * H), *X1 = ensure(d_cvx1, Tf * H), *Y = ensure(d_cvy, Tf * H), *QKV = ensure(d_cvqkv, Tf * 3 * H);
  float *AO = ensure(d_cvao, Tf * std::max(H, C)), *FF = ensure(d_cvff, Tf * Fh);
  const dim3 lg((maxF + CVL_WARPS - 1) / CVL_WARPS, B), lb(32 * CVL_WARPS);
  // precision modes >= 1: the projection and the transformer's qkv / out / FFN convs on conv_tc_kernel, attention on
  // attn_tc_kernel; every producer of a GEMM operand also writes its split-bf16 planes.  All of
  // them are 1x1, and the attention masks keys past a clip, so no plane row behind a clip is read (no tail zeroing).
  Planes PX, P512, PQKV, PAO, PX1, PFF;
  if (cv_tc) {
    P512 = planes(50, (long)Tf, 1, C); PX = planes(51, (long)Tf, 1, H); PQKV = planes(52, (long)Tf, 1, 3 * H);
    PAO = planes(53, (long)Tf, 1, H); PX1 = planes(54, (long)Tf, 1, H); PFF = planes(55, (long)Tf, 1, Fh);
  }
  auto ln = [&](const float* a, const float* yy, const float* g, const float* bt, float* o, const int* oo, int width, const Planes* pl) {
    klaunch(cv_ln_kernel, lg, lb, (size_t)0, a, yy, g, bt, c.cv_ln_eps, o, Lf, Of, oo, width, pl ? pl->hi : (__nv_bfloat16*)nullptr,
            pl ? pl->lo : (__nv_bfloat16*)nullptr);
    CK(cudaGetLastError());
    ++launches;
  };
  auto gemm = [&](const Planes& in, const TcW& w, const ConvW& cw, float* y, const float* res, const Planes* out, int epi) {
    TcSpec s;
    s.in = in; s.w = w; s.bias = cw.b; s.Cin = cw.Cin; s.Cout = cw.Cout;
    s.y = y; s.ldy = cw.Cout; s.res = res; s.ldr = res ? cw.Cout : 0; s.epi = epi;
    if (out) s.out = *out;
    launch_tc({s}, 1, Lf, Of, maxF, B);
  };
  ln(x, nullptr, cv_fp_g, cv_fp_b, AO, Of, C, cv_tc ? &P512 : nullptr);
  if (cv_tc) gemm(P512, cv_tfp, cv_fp, X, nullptr, nullptr, 0);
  else launch_conv({mk(cv_fp, AO, C, 0, X, H, 0, 1, 0)}, 1, Lf, Of, maxF, B);
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
      launch_conv(pp, 1, Lf, Of, maxF, B);
    }
  ln(X, Y, cv_enc_g, cv_enc_b, X1, Of, H, cv_tc ? &PX : nullptr);
  if (debug_flags & 1) CK(cudaMemcpyAsync(ensure(d_cvdbg, Tf * H), X1, Tf * H * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  float *xa = X1, *xb = X;
  for (size_t l = 0; l < cv_enc.size() && cv_tc; ++l) {
    const EncLayerW& Lw = cv_enc[l];
    gemm(PX, Lw.t_qkv, Lw.qkv, QKV, nullptr, &PQKV, 0);
    if (attn_use_tc(Lw, H, Lf, maxF)) launch_attn_tc(PQKV, AO, &PAO, Lw, H, Lf, Of, maxF);
    else launch_attn(QKV, AO, Lw, H, Lf, Of, maxF, &PAO);
    gemm(PAO, Lw.t_o, Lw.o, Y, xa, nullptr, 0);
    ln(Y, nullptr, Lw.ln1.g, Lw.ln1.b, xb, Of, H, &PX1);
    gemm(PX1, Lw.t_ffn1, Lw.ffn1, FF, nullptr, nullptr, 0);
    gelu(FF, Fh, Lf, Of, maxF, &PFF);
    gemm(PFF, Lw.t_ffn2, Lw.ffn2, Y, xb, nullptr, 0);
    if (l + 1 == cv_enc.size()) ln(Y, nullptr, Lw.ln2.g, Lw.ln2.b, out, out_offs ? out_offs : Of, H, nullptr);
    else ln(Y, nullptr, Lw.ln2.g, Lw.ln2.b, xa, Of, H, &PX);
  }
  for (size_t l = 0; l < cv_enc.size() && !cv_tc; ++l) {
    const EncLayerW& Lw = cv_enc[l];
    launch_conv({mk(Lw.qkv, xa, H, 0, QKV, 3 * H, 0, 1, 0)}, 1, Lf, Of, maxF, B);
    launch_attn(QKV, AO, Lw, H, Lf, Of, maxF, nullptr);
    ConvP po = mk(Lw.o, AO, H, 0, Y, H, 0, 1, 0);
    po.res = xa; po.ldr = H;
    launch_conv({po}, 1, Lf, Of, maxF, B);
    ln(Y, nullptr, Lw.ln1.g, Lw.ln1.b, xb, Of, H, nullptr);
    launch_conv({mk(Lw.ffn1, xb, H, 0, FF, Fh, 0, 1, 0)}, 1, Lf, Of, maxF, B);
    gelu(FF, Fh, Lf, Of, maxF, nullptr);
    ConvP p2 = mk(Lw.ffn2, FF, Fh, 0, Y, H, 0, 1, 0);
    p2.res = xb; p2.ldr = H;
    launch_conv({p2}, 1, Lf, Of, maxF, B);
    if (l + 1 == cv_enc.size()) ln(Y, nullptr, Lw.ln2.g, Lw.ln2.b, out, out_offs ? out_offs : Of, H, nullptr);
    else ln(Y, nullptr, Lw.ln2.g, Lw.ln2.b, xa, Of, H, nullptr);
  }
}

// Front end (or the caller's log-mel), the three LSTM layers over every slice, and the embedding.  seq: the slice table of
// d_sseq (host copy); max_len: the longest slice.
void vtts_engine::spk_enqueue(bool from_mel, const std::vector<int>& seq, int max_len) {
  const int ns = spk_nseq;
  int* ds = ensure(d_sseq, seq.size());
  CK(cudaMemcpyAsync(ds, seq.data(), seq.size() * sizeof(int), cudaMemcpyHostToDevice, stream));
  const int *xrow = ds, *slen = ds + ns, *soff = ds + 2 * ns, *last = ds + 3 * ns + 1, *of_clip = ds + 4 * ns + 1;
  vc_upload(from_mel, false);
  const float* feat = front_end(from_mel);
  // Sequences per cluster: the fewest that keep every cluster co-resident; more sequences per cluster lengthen each step,
  // more clusters than fit run in waves.
  int NS = 1, li = 0;
  while (NS < 8 && (ns + NS - 1) / NS > spk_clusters[li]) { NS *= 2; ++li; }
  const int groups = (ns + NS - 1) / NS;
  // The projections run with one fixed launch shape (no split-K across CTAs or thread groups), so every row is summed in the
  // same order whatever the batch: a clip's g does not depend on the clips it is batched with.  Layers 1 and 2 launch over
  // the slices, so the host-side lengths the launch heuristics read are the slices' for those launches.
  struct Saved {
    vtts_engine* e; int ms, ming, bigg, autog; std::vector<int> vf, hf;
    explicit Saved(vtts_engine* h) : e(h), ms(h->conv_max_s), ming(h->conv_min_g), bigg(h->conv_big_g), autog(h->conv_auto_g),
                                     vf(h->v_frm_len), hf(h->h_frm_len) {}
    ~Saved() { e->conv_max_s = ms; e->conv_min_g = ming; e->conv_big_g = bigg; e->conv_auto_g = autog; e->v_frm_len = vf; e->h_frm_len = hf; }
  } saved(this);
  conv_max_s = 1; conv_min_g = 1; conv_big_g = 1; conv_auto_g = 0;
  const std::vector<int> slen_h(seq.begin() + ns, seq.begin() + 2 * ns);
  const float* x = feat;
  for (int l = 0; l < 3; ++l) {
    if (l == 1) { v_frm_len = slen_h; h_frm_len = slen_h; }
    float* xp = ensure(d_sx[l], (size_t)(l == 0 ? Tfrm : spk_rows) * SPK_GATES);
    float* hs = ensure(d_sh[l], (size_t)spk_rows * SPK_H);
    if (l == 0) launch_conv({mk(spk_ih[0], x, spec_pad, 0, xp, SPK_GATES, 0, 1, 0)}, 1, d_frm_len.p, d_frm_off.p, maxFrm, B);
    else launch_conv({mk(spk_ih[l], x, SPK_H, 0, xp, SPK_GATES, 0, 1, 0)}, 1, slen, soff, max_len, ns);
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
// Pinned staging of one call (fixed layout for a given batch / length bucket): ints [frm_len B][frm_off B+1][identity B],
// prm[16], unit rows [Tfrm][QV_UNITS] (clips packed as the engine's rows, SEQ_GAP zero rows between them), g [B][gin],
// eps [B][inter][maxFrm].
vtts_engine::QvPin vtts_engine::qv_layout(bool eps) {
  const vtts_config& c = cfg;
  const size_t ints = (size_t)(3 * B + 1) * sizeof(int);
  const size_t head = (ints + 63) / 64 * 64;
  const size_t nu = (size_t)Tfrm * QV_UNITS, ng = (size_t)B * c.gin_channels, ne = eps ? (size_t)B * c.inter_channels * maxFrm : 0;
  char* pin = ensure_pinned(h_pin_qv, head + (16 + nu + ng + ne) * sizeof(float) + 64);
  QvPin pp;
  pp.frm_len = reinterpret_cast<int*>(pin);
  pp.frm_off = pp.frm_len + B;
  pp.ident = pp.frm_off + B + 1;
  pp.prm = reinterpret_cast<float*>(pin + head);
  pp.units = pp.prm + 16;
  pp.g = pp.units + nu;
  pp.eps = pp.g + ng;
  return pp;
}

void vtts_engine::quickvc_enqueue(bool eps, bool from_wav) {
  const vtts_config& c = cfg;
  const int I = c.inter_channels, G = c.gin_channels;
  if (!capturing) CK(cudaEventRecord(ev[4], stream));
  QvPin pp = qv_layout(eps);
  int* fl = ensure(d_frm_len, B);
  int* fo = ensure(d_frm_off, B + 1);
  int* ident = ensure(d_vint, B);
  float* prm = ensure(d_vprm, 16);
  float* units = ensure(d_units, (size_t)Tfrm * QV_UNITS);
  float* g = ensure(d_qg, (size_t)B * G);
  CK(cudaMemcpyAsync(fl, pp.frm_len, B * sizeof(int), cudaMemcpyHostToDevice, stream));
  CK(cudaMemcpyAsync(fo, pp.frm_off, (B + 1) * sizeof(int), cudaMemcpyHostToDevice, stream));
  CK(cudaMemcpyAsync(ident, pp.ident, B * sizeof(int), cudaMemcpyHostToDevice, stream));
  CK(cudaMemcpyAsync(prm, pp.prm, 16 * sizeof(float), cudaMemcpyHostToDevice, stream));
  if (from_wav) {      // ContentVec writes the unit rows; the gaps between clips and the bucket's tail stay zero
    CK(cudaMemsetAsync(units, 0, (size_t)Tfrm * QV_UNITS * sizeof(float), stream));
    cv_enqueue(units, fo);
  } else {
    CK(cudaMemcpyAsync(units, pp.units, (size_t)Tfrm * QV_UNITS * sizeof(float), cudaMemcpyHostToDevice, stream));
  }
  CK(cudaMemcpyAsync(g, pp.g, (size_t)B * G * sizeof(float), cudaMemcpyHostToDevice, stream));
  float* noise = nullptr;
  if (eps) {
    noise = ensure(d_vnoise, (size_t)B * I * maxFrm);
    CK(cudaMemcpyAsync(noise, pp.eps, (size_t)B * I * maxFrm * sizeof(float), cudaMemcpyHostToDevice, stream));
  }
  // ---- g's cond rows [B][condR] (the flow's WN cond layers, then dec.cond) in d_condv: the uploaded g rows are the table
  //      cond_vc_kernel reads, through the identity index
  float* cond = ensure(d_condv, (size_t)B * condR);
  klaunch(cond_vc_kernel, dim3((condR + 7) / 8, B), dim3(256), (size_t)(G * sizeof(float)), (const float*)g, (const int*)ident, cond_w,
          cond_b, condR, (const float*)nullptr, (const float*)nullptr, 0, cond, (float*)nullptr, G, B, B);
  CK(cudaGetLastError());
  ++launches;
  // ---- z_p, m_p, logs_p = enc_p(c)   (models.py:868)
  posterior_encode(units, QV_UNITS, noise, nullptr, 0);
  // ---- z = flow(z_p, g, reverse=True)   (models.py:869)
  float* z = d_z.p;
  const bool flow_on_tc = tc && !flow.empty() && !flow[0].t_in.empty();
  if (flow_on_tc) flow_tc(z, fl, fo, false, cond, condR, /*forward=*/false);
  else flow_ffma(z, fl, fo, cond, condR, /*forward=*/false);
  if (!capturing) CK(cudaEventRecord(ev[5], stream));
  // ---- o = dec(z * c_mask, g)   (models.py:870)
  decode(z, fl, fo);
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
    h->err = h->cfg.model_family == VTTS_FAMILY_QUICKVC ? "this entry point serves VITS2 models; the engine holds a QuickVC model"
                                                        : "this entry point serves QuickVC models; the engine holds a VITS2 model";
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

void setup_lengths(vtts_handle h, const int64_t* lengths, int B, int t_max) {
  REQUIRE(B >= 1 && B <= 16384 && t_max >= 1, VTTS_ERR_INVALID, "bad batch size / t_max");
  h->B = B;
  h->h_tok_len.resize(B);
  h->h_tok_off.resize(B + 1);
  int off = 0, mx = 0;
  for (int b = 0; b < B; ++b) {
    REQUIRE(lengths[b] >= 1 && lengths[b] <= t_max, VTTS_ERR_INVALID, "input_lengths must be in [1, t_max]");
    h->h_tok_len[b] = (int)lengths[b];
    h->h_tok_off[b] = off;
    off += (int)lengths[b] + (b + 1 < B ? SEQ_GAP : 0);
    mx = std::max(mx, (int)lengths[b]);
  }
  h->h_tok_off[B] = off;
  (void)mx;
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
  std::vector<int> packed(h->Ttok), sid32(B);
  for (int b = 0; b < B; ++b) {
    for (int t = 0; t < h->h_tok_len[b]; ++t) {
      const int64_t id = ids[(size_t)b * t_max + t];
      REQUIRE(id >= 0 && id < h->cfg.n_vocab, VTTS_ERR_INVALID, "phoneme id out of range [0, n_vocab)");
      packed[h->h_tok_off[b] + t] = (int)id;
    }
    REQUIRE(!h->has_g || (sid[b] >= 0 && sid[b] < h->cfg.n_speakers), VTTS_ERR_INVALID, "speaker id out of range [0, n_speakers)");
    sid32[b] = (int)sid[b];
  }
  h->stage1(packed.data(), sid32.data(), t_max, noise_dp);
  h->run_graphed({0x11, B, h->maxTok, h->Ttok, noise_dp ? 1 : 0}, [&] { h->phase1(packed.data(), nullptr, t_max, nullptr, sid32.data(), noise_dp, false); });
}

static void impl_durations(vtts_handle h, const int64_t* ids, const int64_t* lengths, const int64_t* sid, int B, int t_max,
                   const float* scales, const float* noise_dp, uint64_t seed, int64_t* y_lengths, int32_t* durations) {
  enqueue_phase1_host(h, ids, lengths, sid, B, t_max, scales, noise_dp, seed, false);
  h->finish1();
  if (B == 1) h->spec_learn();
  for (int b = 0; b < B; ++b) y_lengths[b] = h->h_frm_len[b];
  if (durations) {
    std::vector<int> wc(h->Ttok);
    CK(cudaMemcpyAsync(wc.data(), h->d_wceil.p, h->Ttok * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
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
  h->run_graphed({0x22, h->B, h->maxFrm, h->Tfrm, noise_z ? 1 : 0}, [&] { h->phase2(noise_z, z_ld, false); });
  const size_t nw = (size_t)h->real_Tfrm * h->hop;
  char* pin = h->ensure_pinned((size_t)h->Tfrm * h->hop * sizeof(float) + (size_t)h->Tfrm * sizeof(int) + 64);
  float* pw = reinterpret_cast<float*>(pin);
  int* pi = reinterpret_cast<int*>(pw + (size_t)h->Tfrm * h->hop);
  CK(cudaMemcpyAsync(pw, h->d_wav.p, nw * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  if (frame_token) CK(cudaMemcpyAsync(pi, h->d_ftok.p, (size_t)h->real_Tfrm * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaEventRecord(h->ev[7], h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (int b = 0; b < h->B; ++b) {
    memcpy(wav + (size_t)b * wav_ld, pw + (size_t)h->h_frm_off[b] * h->hop, (size_t)h->h_frm_len[b] * h->hop * sizeof(float));
    if (frame_token) memcpy(frame_token + (size_t)b * idx_ld, pi + h->h_frm_off[b], (size_t)h->h_frm_len[b] * sizeof(int));
  }
  collect_timings(h);
  h->have_durations = false;
}

static void enqueue_phase1_dev(vtts_handle h, const int64_t* d_ids, const int64_t* lengths_host, const int64_t* d_sid, int B, int t_max,
                              const float* scales, const float* d_noise_dp, uint64_t seed, bool may_speculate) {
  setup_lengths(h, lengths_host, B, t_max);
  memcpy(h->scales, scales, 3 * sizeof(float));
  h->seed = seed;
  h->spec_cap = (may_speculate && spec_ok(h, B)) ? vtts_engine::bucket_frm(h->spec_predict()) : 0;
  h->stage1(nullptr, nullptr, t_max, nullptr);
  h->eps_dp_ld = t_max;      // device noise is read in the caller's [B][2][t_max] layout
  h->run_graphed({0x33, B, h->maxTok, h->Ttok, t_max, (long long)(uintptr_t)d_ids, (long long)(uintptr_t)d_sid, (long long)(uintptr_t)d_noise_dp},
                 [&] { h->phase1(nullptr, d_ids, t_max, d_sid, nullptr, d_noise_dp, true); });
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
    h->run_graphed({0x22, h->B, h->maxFrm, h->Tfrm, noise_z ? 1 : 0}, [&] { h->phase2(noise_z, z_ld, false); });
    // the true length is not known on the host yet: the bucket's worth of samples comes back
    const size_t ncap = (size_t)cap * h->hop;
    char* pin = h->ensure_pinned(ncap * sizeof(float) + (size_t)cap * sizeof(int) + 64);
    float* pw = reinterpret_cast<float*>(pin);
    int* pi = reinterpret_cast<int*>(pw + ncap);
    CK(cudaMemcpyAsync(pw, h->d_wav.p, ncap * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    if (frame_token) CK(cudaMemcpyAsync(pi, h->d_ftok.p, (size_t)cap * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
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
      memcpy(wav, pw, (size_t)real * h->hop * sizeof(float));
      if (frame_token) memcpy(frame_token, pi, (size_t)real * sizeof(int));
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
    h->run_graphed({0x44, h->B, h->maxFrm, h->Tfrm, z_ld, (long long)(uintptr_t)d_noise_z}, [&] { h->phase2(d_noise_z, z_ld, true); });
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
      REQUIRE(L > h->vc_pad, VTTS_ERR_INVALID, "clip too short: the reflect padding of the spectrogram needs more than " +
              std::to_string(h->vc_pad) + " samples");
      REQUIRE(L < (1LL << 30), VTTS_ERR_INVALID, "clip too long");
      frames[b] = (int)((L + 2 * h->vc_pad - c.filter_length) / c.hop_length + 1);
    }
  }
  return frames;
}

// Sets the frame shape and stages the recordings, speaker ids (sid_tgt may be null), noise and scalars in vc_layout.
static void stage_clips(vtts_handle h, bool from_spec, const float* in, const int64_t* lengths, int64_t ld, const std::vector<int>& frames,
                        const int64_t* sid_src, const int64_t* sid_tgt, float noise_scale, const float* noise_q, int q_ld, uint64_t seed) {
  const vtts_config& c = h->cfg;
  const int B = h->B;
  h->h_frm_len = frames;
  h->h_frm_off.assign(B + 1, 0);
  int off = 0;
  for (int b = 0; b < B; ++b) { h->h_frm_off[b] = off; off += frames[b] + (b + 1 < B ? SEQ_GAP : 0); }
  h->h_frm_off[B] = off;
  h->set_frame_shape();
  h->vc_wld = (h->maxFrm + 2) * c.hop_length + c.filter_length;
  const int maxF = h->maxFrm, I = c.inter_channels, C = c.spec_channels;
  vtts_engine::VcPin pp = h->vc_layout(from_spec, noise_q != nullptr);
  memcpy(pp.frm_len, frames.data(), B * sizeof(int));
  memcpy(pp.frm_off, h->h_frm_off.data(), (B + 1) * sizeof(int));
  for (int b = 0; b < B; ++b) {
    pp.clip_len[b] = (int)lengths[b];
    pp.sid[b] = sid_src ? (int)sid_src[b] : 0;
    pp.sid[B + b] = sid_tgt ? (int)sid_tgt[b] : 0;
    if (from_spec) {
      for (int ch = 0; ch < C; ++ch)
        memcpy(pp.in + ((size_t)b * C + ch) * maxF, in + ((size_t)b * C + ch) * ld, (size_t)frames[b] * sizeof(float));
    } else {
      memcpy(pp.in + (size_t)b * h->vc_wld, in + (size_t)b * ld, (size_t)lengths[b] * sizeof(float));
    }
    if (noise_q)
      for (int ch = 0; ch < I; ++ch)
        memcpy(pp.eps + ((size_t)b * I + ch) * maxF, noise_q + ((size_t)b * I + ch) * q_ld, (size_t)frames[b] * sizeof(float));
  }
  for (int i = 0; i < 16; ++i) pp.prm[i] = 0.f;
  pp.prm[0] = noise_scale;
  const uint32_t lo = (uint32_t)seed, hi = (uint32_t)(seed >> 32);
  memcpy(&pp.prm[4], &lo, 4);
  memcpy(&pp.prm[5], &hi, 4);
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
  h->run_graphed({0x55, B, h->maxFrm, h->Tfrm, from_spec ? 1 : 0, noise_q ? 1 : 0},
                 [&] { h->convert_enqueue(from_spec, noise_q != nullptr); });
  const size_t nw = (size_t)h->real_Tfrm * h->hop;
  float* pw = reinterpret_cast<float*>(h->ensure_pinned((size_t)h->Tfrm * h->hop * sizeof(float) + 64));
  CK(cudaMemcpyAsync(pw, h->d_wav.p, nw * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaEventRecord(h->ev[7], h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (int b = 0; b < B; ++b) {
    memcpy(out_wav + (size_t)b * out_ld, pw + (size_t)h->h_frm_off[b] * h->hop, (size_t)frames[b] * h->hop * sizeof(float));
    out_frames[b] = frames[b];
  }
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
  float* pg = reinterpret_cast<float*>(h->ensure_pinned((size_t)B * SPK_H * sizeof(float) + 64));
  CK(cudaMemcpyAsync(pg, h->d_sg.p, (size_t)B * SPK_H * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  memcpy(g_out, pg, (size_t)B * SPK_H * sizeof(float));
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
    for (int64_t t = 0; t < tx; ++t) {
      const int64_t id = ids[(size_t)b * t_max + t];
      REQUIRE(id >= 0 && id < c.n_vocab, VTTS_ERR_INVALID, "phoneme id out of range [0, n_vocab)");
    }
    REQUIRE(!h->has_g || (sid && sid[b] >= 0 && sid[b] < c.n_speakers), VTTS_ERR_INVALID, "speaker id out of range [0, n_speakers)");
  }
  const int real_max = *std::max_element(frames.begin(), frames.end());
  REQUIRE(!token_of_frame || tof_ld >= real_max, VTTS_ERR_CAPACITY, "tof_ld is smaller than max(frames)");
  REQUIRE(!noise_q || q_ld >= real_max, VTTS_ERR_CAPACITY, "noise_q has fewer columns than max(frames)");
  setup_lengths(h, id_lengths, B, t_max);
  stage_clips(h, from_spec, in, lengths, ld, frames, h->has_g ? sid : nullptr, nullptr, noise_scale, noise_q, q_ld, seed);
  {
    vtts_engine::P1Pin pp = h->p1_layout(t_max, false);
    memcpy(pp.len, h->h_tok_len.data(), B * sizeof(int));
    memcpy(pp.off, h->h_tok_off.data(), (B + 1) * sizeof(int));
    memset(pp.ids, 0, (size_t)h->Ttok * sizeof(int));
    for (int b = 0; b < B; ++b)
      for (int t = 0; t < h->h_tok_len[b]; ++t) pp.ids[h->h_tok_off[b] + t] = (int)ids[(size_t)b * t_max + t];
  }
  h->run_graphed({0x66, B, h->maxTok, h->Ttok, h->maxFrm, h->Tfrm, from_spec ? 1 : 0, noise_q ? 1 : 0},
                 [&] { h->align_enqueue(from_spec, noise_q != nullptr); });
  const size_t nt = (size_t)h->real_Ttok, nf = (size_t)h->real_Tfrm;
  int* pin = reinterpret_cast<int*>(h->ensure_pinned((nt + nf + (size_t)B) * sizeof(int) + 64));
  CK(cudaMemcpyAsync(pin, h->d_adur.p, nt * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(pin + nt, h->d_atof.p, nf * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(pin + nt + nf, h->d_ascore.p, (size_t)B * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaEventRecord(h->ev[7], h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (int b = 0; b < B; ++b) {
    const int tx = h->h_tok_len[b], ty = frames[b];
    int32_t* d = durations + (size_t)b * t_max;
    memcpy(d, pin + h->h_tok_off[b], (size_t)tx * sizeof(int));
    std::fill(d + tx, d + t_max, 0);
    if (token_of_frame) {
      int32_t* f = token_of_frame + (size_t)b * tof_ld;
      memcpy(f, pin + nt + h->h_frm_off[b], (size_t)ty * sizeof(int));
      std::fill(f + ty, f + tof_ld, -1);
    }
    if (score) memcpy(score + b, pin + nt + nf + b, sizeof(float));
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
  h->run_graphed({0xC7, B, h->cvp.maxS, h->cvp.tot0}, [&] { h->cv_enqueue(h->ensure(h->d_cvu, Tf * H), nullptr); });
  float* pu = reinterpret_cast<float*>(h->ensure_pinned(Tf * H * sizeof(float) + 64));
  CK(cudaMemcpyAsync(pu, h->d_cvu.p, Tf * H * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (int b = 0; b < B; ++b) {
    const size_t n = (size_t)frames[b] * H;
    float* dst = units + (size_t)b * units_ld * H;
    memcpy(dst, pu + (size_t)h->cvp.h[(NL + NL - 1) * B + b] * H, n * sizeof(float));
    std::fill(dst + n, dst + (size_t)units_ld * H, 0.f);
    out_frames[b] = frames[b];
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
  h->h_frm_len = frames;
  h->h_frm_off.assign(B + 1, 0);
  int off = 0;
  for (int b = 0; b < B; ++b) { h->h_frm_off[b] = off; off += frames[b] + (b + 1 < B ? SEQ_GAP : 0); }
  h->h_frm_off[B] = off;
  h->set_frame_shape();
  const int maxF = h->maxFrm, I = c.inter_channels, G = c.gin_channels;
  vtts_engine::QvPin pp = h->qv_layout(noise != nullptr);
  memcpy(pp.frm_len, frames.data(), B * sizeof(int));
  memcpy(pp.frm_off, h->h_frm_off.data(), (B + 1) * sizeof(int));
  for (int b = 0; b < B; ++b) {
    pp.ident[b] = b;
    const int o = h->h_frm_off[b];
    if (units) {
    memcpy(pp.units + (size_t)o * vtts_engine::QV_UNITS, units + (size_t)b * units_ld * vtts_engine::QV_UNITS,
           (size_t)frames[b] * vtts_engine::QV_UNITS * sizeof(float));
    const int gap_end = b + 1 < B ? h->h_frm_off[b + 1] : h->Tfrm;       // rows behind the clip: the gap, or the bucket's tail
    memset(pp.units + (size_t)(o + frames[b]) * vtts_engine::QV_UNITS, 0, (size_t)(gap_end - o - frames[b]) * vtts_engine::QV_UNITS * sizeof(float));
    }
    memcpy(pp.g + (size_t)b * G, g + (size_t)b * G, G * sizeof(float));
    if (noise)
      for (int ch = 0; ch < I; ++ch)
        memcpy(pp.eps + ((size_t)b * I + ch) * maxF, noise + ((size_t)b * I + ch) * noise_ld, (size_t)frames[b] * sizeof(float));
  }
  for (int i = 0; i < 16; ++i) pp.prm[i] = 0.f;
  pp.prm[0] = noise_scale;
  const uint32_t lo = (uint32_t)seed, hi = (uint32_t)(seed >> 32);
  memcpy(&pp.prm[4], &lo, 4);
  memcpy(&pp.prm[5], &hi, 4);
  if (wav)
    h->run_graphed({0x78, B, h->maxFrm, h->Tfrm, noise ? 1 : 0, h->cvp.maxS, h->cvp.tot0}, [&] { h->quickvc_enqueue(noise != nullptr, true); });
  else
    h->run_graphed({0x77, B, h->maxFrm, h->Tfrm, noise ? 1 : 0}, [&] { h->quickvc_enqueue(noise != nullptr); });
  const size_t nw = (size_t)h->real_Tfrm * h->hop;
  float* pw = reinterpret_cast<float*>(h->ensure_pinned((size_t)h->Tfrm * h->hop * sizeof(float) + 64));
  CK(cudaMemcpyAsync(pw, h->d_wav.p, nw * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaEventRecord(h->ev[7], h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (int b = 0; b < B; ++b) {
    const size_t n = (size_t)frames[b] * h->hop;
    memcpy(out_wav + (size_t)b * out_ld, pw + (size_t)h->h_frm_off[b] * h->hop, n * sizeof(float));
    std::fill(out_wav + (size_t)b * out_ld + n, out_wav + (size_t)(b + 1) * out_ld, 0.f);
    out_frames[b] = frames[b];
  }
}

static void impl_synthesize_dev(vtts_handle h, const float* d_noise_z, int z_ld, float* d_wav, int64_t wav_ld) {
  REQUIRE(h->have_durations, VTTS_ERR_STATE, "vtts_synthesize_dev called without vtts_durations_dev");
  REQUIRE((int64_t)h->real_maxFrm * h->hop <= wav_ld, VTTS_ERR_CAPACITY, "wav_ld is smaller than hop * max(y_lengths)");
  REQUIRE(!d_noise_z || z_ld >= h->real_maxFrm, VTTS_ERR_CAPACITY, "noise_z has fewer columns than max(y_lengths)");
  h->run_graphed({0x44, h->B, h->maxFrm, h->Tfrm, z_ld, (long long)(uintptr_t)d_noise_z}, [&] { h->phase2(d_noise_z, z_ld, true); });
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
    CK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    for (auto& st : h->side) CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    for (auto& e : h->ev_join) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    for (auto& e : h->ev) CK(cudaEventCreate(&e));
    h->blob_floats = blob_floats;
    CK(cudaMalloc(&h->d_blob, blob_floats * sizeof(float)));
    CK(cudaMemcpyAsync(h->d_blob, blob, blob_floats * sizeof(float), blob_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, h->stream));
    std::istringstream is(manifest);
    std::string name;
    unsigned long long off, n;
    while (is >> name >> off >> n) {
      REQUIRE(off + n <= blob_floats, VTTS_ERR_WEIGHTS, "manifest entry exceeds the blob");
      h->tensors[name] = Tensor{h->d_blob + off, (size_t)n};
    }
    if (const char* e = getenv("VTTS_CONV_MAXS")) h->conv_max_s = std::max(1, atoi(e));
    if (const char* e = getenv("VTTS_CONV_TARGET")) h->conv_target = std::max(1, atoi(e));
    if (const char* e = getenv("VTTS_CONV_MAXG")) h->conv_max_g = std::max(1, std::min(4, atoi(e)));
    if (const char* e = getenv("VTTS_CONV_BIGG")) h->conv_big_g = std::max(1, std::min(4, atoi(e)));   // thread groups per CTA on machine-filling FFMA launches
    if (const char* e = getenv("VTTS_TC_TALL")) h->tc_tall = atoi(e);
    if (const char* e = getenv("VTTS_TC_BASEOFF")) h->tc_baseoff = atoi(e);
    if (const char* e = getenv("VTTS_TC_BN")) h->tc_bn = atoi(e);
    if (const char* e = getenv("VTTS_TC_MULTICAST")) h->tc_mc = atoi(e);
    if (const char* e = getenv("VTTS_TC_SPLIT")) h->tc_split = atoi(e);
    if (const char* e = getenv("VTTS_TC_MINSTEPS")) h->tc_min_steps = std::max(1, atoi(e));   // k-steps per CTA below which split-K stops
    if (const char* e = getenv("VTTS_TC_PERSIST")) h->tc_persist = atoi(e);                 // 0: one tile per CTA also on machine-filling launches; 2: persistent grid on every launch without split-K (tests)
    if (const char* e = getenv("VTTS_TC_DBGSKIP")) h->tc_dbgskip = atoi(e);                 // timing experiments only (wrong results)
    if (const char* e = getenv("VTTS_TC_WMC")) h->tc_wmc = atoi(e);                         // 1: weight-tile multicast between CTA pairs of persistent launches (measured neutral, off)
    if (const char* e = getenv("VTTS_TC_PERSIST_MIN")) h->tc_persist_min = std::max(1, atoi(e));   // tiles per SM from which the persistent grid is used
    if (const char* e = getenv("VTTS_MRF_BRANCH")) h->mrf_branch = atoi(e);
    if (const char* e = getenv("VTTS_MRF_HEAVY_FIRST")) h->mrf_heavy_first = atoi(e);
    if (const char* e = getenv("VTTS_ATTN_SPLIT")) h->attn_split = atoi(e);       // 0: never use the split-KV attention
    if (const char* e = getenv("VTTS_CONV_AUTOG")) h->conv_auto_g = std::max(0, atoi(e));   // k-steps per rank needed to add thread groups; 0 = never
    if (const char* e = getenv("VTTS_CONV_MING")) h->conv_min_g = std::max(1, std::min(4, atoi(e)));      // 0 auto, 1 off, 2/4/8 cap
    if (const char* e = getenv("VTTS_ATTN_ROWS")) h->attn_rows = atoi(e);
    if (const char* e = getenv("VTTS_ATTN_TC")) h->attn_tc_mode = atoi(e);
    if (const char* e = getenv("VTTS_PDL")) h->use_pdl = atoi(e) != 0;
    if (const char* e = getenv("VTTS_NO_POLL")) h->use_poll = atoi(e) == 0;
    if (const char* e = getenv("VTTS_NO_GRAPHS")) h->use_graphs = atoi(e) == 0;
    if (const char* e = getenv("VTTS_BUCKETS")) h->use_buckets = atoi(e) != 0;
    if (const char* e = getenv("VTTS_SPEC")) h->use_spec = atoi(e) != 0;
    if (const char* e = getenv("VTTS_SPEC_MARGIN")) h->spec_margin = (float)atof(e);      // (< 1 forces mispredictions: tests)
    if (const char* e = getenv("VTTS_CAPTURE_FIRST")) h->capture_on_first = atoi(e) != 0;   // 0: capture a bucket's graph on its second call          // 0: never enqueue phase 2 before the lengths are known    // 0: size everything by the exact lengths
    if (const char* e = getenv("VTTS_PREFETCH")) h->use_prefetch = atoi(e) != 0;
    REQUIRE(cfg->model_family == VTTS_FAMILY_VITS2 || cfg->model_family == VTTS_FAMILY_QUICKVC, VTTS_ERR_INVALID, "unknown model family");
    if (cfg->model_family == VTTS_FAMILY_QUICKVC) h->bind_quickvc();
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
    CK(cudaStreamSynchronize(h->stream));
  }, G_ATOMIC, ANY_FAMILY);
}

void vtts_destroy(vtts_handle h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  auto fr = [](void* p) { if (p) cudaFree(p); };
  fr(h->d_blob);
  Buf<int>* ib[] = {&h->d_ids, &h->d_tok_len, &h->d_tok_off, &h->d_sid, &h->d_wceil, &h->d_cum, &h->d_frm_len, &h->d_frm_off, &h->d_ftok, &h->d_done_ctr, &h->d_frm_len_real};
  for (auto* b : ib) fr(b->p);
  Buf<float>* fb[] = {&h->d_condv, &h->d_x, &h->d_xb, &h->d_qkv, &h->d_ao, &h->d_y, &h->d_ffh, &h->d_stats, &h->d_dA, &h->d_dB, &h->d_dx,
                      &h->d_h29, &h->d_za, &h->d_zb, &h->d_eps_dp, &h->d_z, &h->d_h, &h->d_h1, &h->d_wx, &h->d_acts, &h->d_skip, &h->d_fqkv,
                      &h->d_fao, &h->d_fy, &h->d_ffh2, &h->d_eps_z, &h->d_d0, &h->d_post, &h->d_wav};
  for (auto* b : fb) fr(b->p);
  Buf<float>* vb[] = {&h->d_vprm, &h->d_vin, &h->d_vlin, &h->d_vfeat, &h->d_vstats, &h->d_vcsrc, &h->d_vnoise, &h->d_vz_dbg, &h->d_vzp_dbg,
                      &h->d_sx[0], &h->d_sx[1], &h->d_sx[2], &h->d_sh[0], &h->d_sh[1], &h->d_sh[2], &h->d_sg, &h->d_units, &h->d_qg,
                      &h->d_cvzero, &h->d_cvwav, &h->d_cvps, &h->d_cvpq, &h->d_cvl[0], &h->d_cvl[1], &h->d_cvx, &h->d_cvx1, &h->d_cvy,
                      &h->d_cvqkv, &h->d_cvao, &h->d_cvff, &h->d_cvu, &h->d_cvdbg};
  for (auto* b : vb) fr(b->p);
  fr(h->d_vint.p);
  fr(h->d_sseq.p);
  fr(h->d_cvi.p);
  for (auto& b : h->d_stage) fr(b.p);
  for (auto& v : h->d_xj) for (auto& b : v) fr(b.p);
  for (auto& v : h->d_tmp) for (auto& b : v) fr(b.p);
  for (Buf<char>* hb : {&h->h_pin, &h->h_pin_in, &h->h_pin_len, &h->h_pin_z, &h->h_pin_vc, &h->h_pin_qv, &h->h_pin_cv}) if (hb->p) cudaFreeHost(hb->p);
  for (auto& kv : h->graphs) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
  fr(h->d_prm.p);
  fr(h->d_pref.p);
  fr(h->d_chunk.p);
  fr(h->d_zp_dbg.p);
  if (h->h_map) cudaFreeHost(h->h_map);
  for (auto& e : h->ev) if (e) cudaEventDestroy(e);
  for (auto& e : h->prof_ev) if (e) cudaEventDestroy(e);
  for (auto& e : h->tc_prof_ev) if (e) cudaEventDestroy(e);
  for (auto& b : h->pl_pool) fr(b.p);
  for (auto& st : h->side) if (st) cudaStreamDestroy(st);
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  for (auto& e : h->ev_join) if (e) cudaEventDestroy(e);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
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
  float* dv = nullptr; int *dp = nullptr, *dl = nullptr;
  const size_t n = (size_t)B * T_y * T_x;
  int rc = VTTS_OK;
  cudaError_t e = cudaSetDevice(device);
  if (e == cudaSuccess) e = cudaMalloc(&dv, n * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&dp, n * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&dl, (size_t)2 * B * sizeof(int));
  if (e == cudaSuccess) e = cudaMemcpy(dv, neg_cent, n * sizeof(float), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(dl, t_ys, (size_t)B * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(dl + B, t_xs, (size_t)B * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) rc = mas_launch(dv, dl, dl + B, B, T_y, T_x, dp, 0);
  if (e == cudaSuccess && rc == VTTS_OK) e = cudaMemcpy(path, dp, n * sizeof(int), cudaMemcpyDeviceToHost);
  if (dv) cudaFree(dv);
  if (dp) cudaFree(dp);
  if (dl) cudaFree(dl);
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
    int* pin = reinterpret_cast<int*>(h->ensure_pinned(h->h_pin_len, 64));
    pin[0] = hi - lo; pin[1] = lo; pin[2] = hi;
    CK(cudaMemcpyAsync(dc, pin, 3 * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    // the launch helpers size grids and split-K from the host copies of the lengths: point them at the chunk
    // (the planes keep the full utterance's row count, Tfrm: the chunk is addressed by its absolute rows)
    const std::vector<int> len0 = h->h_frm_len, off0 = h->h_frm_off, v0 = h->v_frm_len;
    const int max0 = h->maxFrm;
    h->h_frm_len.assign(1, hi - lo);
    h->h_frm_off = {lo, hi};
    h->v_frm_len = h->h_frm_len;
    h->maxFrm = hi - lo;
    try {
      h->last_graphed = false;
      h->decode(h->d_z.p, dc, dc + 1);
    } catch (...) {
      h->h_frm_len = len0; h->h_frm_off = off0; h->maxFrm = max0; h->v_frm_len = v0;
      throw;
    }
    h->h_frm_len = len0; h->h_frm_off = off0; h->maxFrm = max0; h->v_frm_len = v0;
    const size_t n = (size_t)(f1 - f0) * h->hop;
    float* pw = reinterpret_cast<float*>(h->ensure_pinned(n * sizeof(float)));
    CK(cudaMemcpyAsync(pw, h->d_wav.p + (size_t)f0 * h->hop, n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    memcpy(wav, pw, n * sizeof(float));
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
    static unsigned long long* d_tl = nullptr;
    CK(cudaStreamSynchronize(h->stream));
    if (enable == 1) {
      if (!d_tl) CK(cudaMalloc(&d_tl, (1 + 2 * 4000) * 8));
      CK(cudaMemset(d_tl, 0, (1 + 2 * 4000) * 8));
      CK(cudaMemcpyToSymbol(g_timeline, &d_tl, sizeof(d_tl)));
    } else if (enable == 0) {
      unsigned long long* z = nullptr;
      CK(cudaMemcpyToSymbol(g_timeline, &z, sizeof(z)));
    } else if (d_tl && out && n_out) {
      std::vector<unsigned long long> hbuf(1 + 2 * 4000);
      CK(cudaMemcpy(hbuf.data(), d_tl, hbuf.size() * 8, cudaMemcpyDeviceToHost));
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
    else if (nm == "cv_enc_in") { src = h->d_cvdbg.p; n = (size_t)h->cvp.tot0 / h->cv_P * c.cv_hidden; }
    else if (nm.rfind("stage", 0) == 0) {
      const int i = atoi(nm.c_str() + 5);
      REQUIRE(i >= 0 && i < (int)h->d_stage.size(), VTTS_ERR_INVALID, "no such stage");
      int rm = 1, ch = c.upsample_initial_channel;
      for (int j = 0; j <= i; ++j) { rm *= c.upsample_rates[j]; ch /= 2; }
      src = h->d_stage[i].p; n = F * rm * ch;
    }
    REQUIRE(src != nullptr, VTTS_ERR_INVALID, "unknown or unallocated debug tensor");
    REQUIRE(n <= max_floats, VTTS_ERR_CAPACITY, "debug buffer too small");
    CK(cudaMemcpyAsync(out, src, n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    *n_out = n;
  }, G_ATOMIC, ANY_FAMILY);
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

int vtts_quickvc_convert_wav(vtts_handle h, const float* wav, const int64_t* wav_lengths, int B, int64_t wav_ld, const float* g,
                             float noise_scale, const float* noise, int noise_ld, uint64_t seed, float* out_wav, int64_t out_ld,
                             int64_t* out_frames) {
  if (!wav || !wav_lengths || !out_wav || !out_frames) return VTTS_ERR_INVALID;
  return guarded(h, [&] { impl_quickvc_convert(h, nullptr, wav, wav_lengths, B, wav_ld, g, noise_scale, noise, noise_ld, seed, out_wav,
                                               out_ld, out_frames); }, G_ATOMIC, VTTS_FAMILY_QUICKVC);
}

// Host copies of a debug hook's arguments on the device (freed on every exit).
struct DebugBufs {
  std::vector<void*> p;
  ~DebugBufs() { for (void* q : p) cudaFree(q); }
  void* up(const void* src, size_t bytes, cudaStream_t s) {
    void* d = nullptr;
    CK(cudaMalloc(&d, std::max<size_t>(bytes, 16)));
    p.push_back(d);
    if (src) CK(cudaMemcpyAsync(d, src, bytes, cudaMemcpyHostToDevice, s));
    return d;
  }
};

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
    // ---- per-call engine state the launch code reads, restored on every exit
    struct Saved {
      vtts_engine* h;
      int B, maxFrm, maxTok, tc_mode, split, arows;
      std::vector<int> fl, tl, vf, vt;
      explicit Saved(vtts_engine* e) : h(e), B(e->B), maxFrm(e->maxFrm), maxTok(e->maxTok), tc_mode(e->attn_tc_mode),
          split(e->attn_split), arows(e->attn_rows), fl(e->h_frm_len), tl(e->h_tok_len), vf(e->v_frm_len), vt(e->v_tok_len) {}
      ~Saved() {
        h->B = B; h->maxFrm = maxFrm; h->maxTok = maxTok; h->attn_tc_mode = tc_mode; h->attn_split = split; h->attn_rows = arows;
        h->h_frm_len = fl; h->h_tok_len = tl; h->v_frm_len = vf; h->v_tok_len = vt;
      }
    } saved(h);
    h->B = B; h->maxFrm = maxLen; h->maxTok = maxLen;
    h->h_frm_len.assign(lens, lens + B); h->h_tok_len = h->h_frm_len;
    h->v_frm_len = ll; h->v_tok_len = ll;           // the heuristics see the launch lengths
    // ---- kernel selection (refused before anything is launched)
    bool use_tc = false;
    switch (kernel) {
      case VTTS_ATTN_AUTO: use_tc = h->attn_use_tc(*L, H, nullptr, maxLen); break;
      case VTTS_ATTN_TC:
        h->attn_tc_mode = 2;
        REQUIRE(h->attn_tc_ok(*L, H), VTTS_ERR_INVALID, "debug_attention: tensor-core attention is not available for this layer (relative tables / window)");
        use_tc = true;
        break;
      case VTTS_ATTN_SPLIT:
        h->attn_split = 1; h->attn_rows = 1;
        REQUIRE(h->attn_split_fits(*L, H, nullptr, maxLen), VTTS_ERR_INVALID, "debug_attention: the split-KV kernel does not fit this launch");
        break;
      case VTTS_ATTN_R1: h->attn_split = 0; h->attn_rows = 1; break;
      case VTTS_ATTN_R4: h->attn_split = 0; h->attn_rows = 4; break;
      default: break;                               // VTTS_ATTN_FFMA: launch_attn's own choice
    }
    REQUIRE(!(use_tc && planes && p_planes != 2), VTTS_ERR_INVALID, "debug_attention: the tensor-core kernel writes 2 output planes");
    // ---- device copies
    DebugBufs dev;
    cudaStream_t st = h->stream;
    CK(cudaStreamSynchronize(st));
    std::vector<int> lo(2 * B + 3);
    for (int b = 0; b < B; ++b) lo[b] = lens[b];
    for (int b = 0; b <= B; ++b) lo[B + b] = (int)off[b];
    lo[2 * B + 1] = (int)rows; lo[2 * B + 2] = 0;   // all rows as one span (input split)
    int* dl = static_cast<int*>(dev.up(lo.data(), lo.size() * sizeof(int), st));
    const int* dlens = dl;
    const int* doffs = dl + B;
    const float* dq = static_cast<const float*>(dev.up(qkv, rows * 3 * H * sizeof(float), st));
    float* dout = static_cast<float*>(dev.up(out, rows * H * sizeof(float), st));   // (the FFMA kernels always write fp32)
    const size_t pn = rows * H;
    Planes po;
    if (planes) {
      __nv_bfloat16* dp = static_cast<__nv_bfloat16*>(dev.up(planes, (size_t)p_planes * pn * 2, st));
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
      if (use_tc) h->launch_attn_tc(pq, out ? dout : nullptr, planes ? &po : nullptr, *L, H, dlens, doffs, maxLen);
      else h->launch_attn(dq, dout, *L, H, dlens, doffs, maxLen, planes ? &po : nullptr);
    };
    once();
    CK(cudaStreamSynchronize(st));
    if (out) CK(cudaMemcpy(out, dout, rows * H * sizeof(float), cudaMemcpyDeviceToHost));
    if (planes) CK(cudaMemcpy(planes, po.hi, (size_t)p_planes * pn * 2, cudaMemcpyDeviceToHost));
    if (report) *report = h->last_attn;
    if (iters > 0 && ms_out) {
      cudaEvent_t e0, e1;
      CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
      CK(cudaEventRecord(e0, st));
      for (int i = 0; i < iters; ++i) once();
      CK(cudaEventRecord(e1, st));
      CK(cudaStreamSynchronize(st));
      float ms = 0.f;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      *ms_out = ms / iters;
      cudaEventDestroy(e0); cudaEventDestroy(e1);
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
    // ---- per-call engine state the launch code reads, restored on every exit
    struct Saved {
      vtts_engine* h;
      int B, maxFrm, knobs[11];
      std::vector<int> fl, fo, vf;
      int* kp[11];
      explicit Saved(vtts_engine* e) : h(e), B(e->B), maxFrm(e->maxFrm), fl(e->h_frm_len), fo(e->h_frm_off), vf(e->v_frm_len),
          kp{&e->tc_bn, &e->tc_split, &e->tc_tall, &e->tc_mc, &e->tc_persist, &e->tc_wmc, &e->tc_min_steps, &e->conv_max_s,
             &e->conv_min_g, &e->conv_max_g, &e->conv_big_g} {
        for (int i = 0; i < 11; ++i) knobs[i] = *kp[i];
      }
      ~Saved() {
        h->B = B; h->maxFrm = maxFrm; h->h_frm_len = fl; h->h_frm_off = fo; h->v_frm_len = vf;
        for (int i = 0; i < 11; ++i) *kp[i] = knobs[i];
      }
    } saved(h);
    if (ov) {
      const int v[11] = {ov->tc_bn, ov->tc_split, ov->tc_tall, ov->tc_mc, ov->tc_persist, ov->tc_wmc, ov->tc_min_steps, ov->conv_max_s,
                         ov->conv_min_g, ov->conv_max_g, ov->conv_big_g};
      for (int i = 0; i < 11; ++i) if (v[i] != VTTS_CONV_KEEP) *saved.kp[i] = v[i];
    }
    h->B = B; h->maxFrm = maxLen;
    h->h_frm_len.assign(lens, lens + B);
    h->h_frm_off.assign(off.begin(), off.end());
    h->v_frm_len = h->h_frm_len;                  // the heuristics see this call's lengths
    // ---- device copies (freed on every exit)
    DebugBufs dev;
    cudaStream_t st = h->stream;
    CK(cudaStreamSynchronize(st));
    std::vector<int> lo(2 * B + 1);
    for (int b = 0; b < B; ++b) lo[b] = lens[b];
    for (int b = 0; b <= B; ++b) lo[B + b] = (int)off[b];
    int* dl = static_cast<int*>(dev.up(lo.data(), lo.size() * sizeof(int), st));
    const int* dlens = dl;
    const int* doffs = dl + B;
    float* dy = y ? static_cast<float*>(dev.up(y, y_n * sizeof(float), st)) : nullptr;
    const float* dres = res ? static_cast<const float*>(dev.up(res, res_n * sizeof(float), st)) : nullptr;
    __nv_bfloat16* dp = any_planes ? static_cast<__nv_bfloat16*>(dev.up(p_out, (size_t)p_planes * p_n * 2, st)) : nullptr;
    __nv_bfloat16 *dp_hi = dp, *dp_mid = (dp && p_planes == 3) ? dp + p_n : nullptr, *dp_lo = dp ? dp + (p_planes - 1) * p_n : nullptr;
    auto cond_of = [&](const vtts_conv_problem& q) {
      return q.cond ? static_cast<const float*>(dev.up(q.cond, (size_t)B * q.cond_ld * sizeof(float), st)) : nullptr;
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
        s.w.hi = static_cast<const __nv_bfloat16*>(dev.up(q.w_hi, wn * 2, st));
        s.w.lo = static_cast<const __nv_bfloat16*>(dev.up(q.w_lo, wn * 2, st));
        if (q.w_mid) s.w.mid = static_cast<const __nv_bfloat16*>(dev.up(q.w_mid, wn * 2, st));
        s.bias = static_cast<const float*>(dev.up(q.bias, (size_t)q.Cout * sizeof(float), st));
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
      h->launch_tc(ps, rmul, dlens, doffs, maxLen, B);
    } else {
      const float* dx = static_cast<const float*>(dev.up(x, x_n * sizeof(float), st));
      std::vector<ConvP> ps;
      for (int i = 0; i < n_problems; ++i) {
        const vtts_conv_problem& q = problems[i];
        ConvW W;
        W.Cin = q.Cin; W.Cout = q.Cout; W.k = q.k; W.ldw = (q.Cout + 3) / 4 * 4;
        W.w = static_cast<const float*>(dev.up(q.w, (size_t)q.k * q.Cin * W.ldw * sizeof(float), st));
        W.b = static_cast<const float*>(dev.up(q.bias, (size_t)W.ldw * sizeof(float), st));
        ConvP p = mk(W, dx, q.ldx, q.xoff, dy, q.ldy, q.yoff, q.dil, q.pad);
        p.cond = cond_of(q); p.cond_ld = q.cond_ld;
        p.res = q.res == 1 ? dres : (q.res == 2 ? dy : nullptr); p.ldr = q.ldr; p.roff = q.roff;
        p.in_extra = q.in_extra; p.reflect = q.reflect; p.out_mul = q.out_mul; p.out_add = q.out_add; p.out_seq_extra = q.out_seq_extra;
        p.pro = q.pro; p.slope = q.slope; p.epi = q.epi; p.alpha = q.alpha;
        if (q.planes_on) { p.p_hi = dp_hi; p.p_lo = dp_lo; p.p_mid = dp_mid; p.ldp = q.ldp; }
        p.pl_slope = q.pl_slope;
        ps.push_back(p);
      }
      h->launch_conv(ps, rmul, dlens, doffs, maxLen, B);
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
    // save state that the launch helpers read
    const int B0 = h->B; const std::vector<int> fl0 = h->h_frm_len, tl0 = h->h_tok_len, vf0 = h->v_frm_len, vt0 = h->v_tok_len;
    h->B = 1; h->h_frm_len.assign(1, rows); h->h_tok_len.assign(1, rows); h->v_frm_len = h->h_frm_len; h->v_tok_len = h->h_tok_len;
    int* dl = nullptr; int* dof = nullptr; float *x = nullptr, *y = nullptr, *w = nullptr, *bias = nullptr;
    __nv_bfloat16 *ph = nullptr, *pl = nullptr, *wh = nullptr, *wl = nullptr;
    const int ldw = (Cout + 3) / 4 * 4;
    CK(cudaMalloc(&dl, 8)); CK(cudaMalloc(&dof, 8));
    const int hl[2] = {rows, rows}, ho[2] = {0, rows};
    CK(cudaMemcpy(dl, hl, 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(dof, ho, 8, cudaMemcpyHostToDevice));
    CK(cudaMalloc(&y, (size_t)rows * Cout * 4)); CK(cudaMalloc(&bias, (size_t)ldw * 4)); CK(cudaMemset(bias, 0, (size_t)ldw * 4));
    if (is_tc) {
      CK(cudaMalloc(&ph, (size_t)rows * Cin * 2)); CK(cudaMalloc(&pl, (size_t)rows * Cin * 2));
      CK(cudaMalloc(&wh, (size_t)k * Cout * Cin * 2)); CK(cudaMalloc(&wl, (size_t)k * Cout * Cin * 2));
      CK(cudaMemset(ph, 0, (size_t)rows * Cin * 2)); CK(cudaMemset(pl, 0, (size_t)rows * Cin * 2));
      CK(cudaMemset(wh, 0, (size_t)k * Cout * Cin * 2)); CK(cudaMemset(wl, 0, (size_t)k * Cout * Cin * 2));
    } else {
      CK(cudaMalloc(&x, (size_t)rows * Cin * 4)); CK(cudaMalloc(&w, (size_t)k * Cin * ldw * 4));
      CK(cudaMemset(x, 0, (size_t)rows * Cin * 4)); CK(cudaMemset(w, 0, (size_t)k * Cin * ldw * 4));
    }
    auto once = [&] {
      if (is_tc) {
        TcSpec q;
        q.in.hi = ph; q.in.lo = pl; q.in.C = Cin; q.in.rows = rows;
        q.w.hi = wh; q.w.lo = wl; q.bias = bias; q.Cin = Cin; q.Cout = Cout; q.k = k; q.dil = dil; q.pad = dil * (k - 1) / 2;
        q.y = y; q.ldy = Cout;
        h->launch_tc({q}, 1, dl, dof, rows, 1);
      } else {
        ConvW W; W.w = w; W.b = bias; W.Cin = Cin; W.Cout = Cout; W.k = k; W.ldw = ldw;
        h->launch_conv({mk(W, x, Cin, 0, y, Cout, 0, dil, dil * (k - 1) / 2)}, 1, dl, dof, rows, 1);
      }
    };
    const bool prof0 = h->profiling; h->profiling = false;
    for (int i = 0; i < 3; ++i) once();
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    // the launches are captured into one CUDA graph so that the host launch path is not what gets timed
    cudaGraph_t graph = nullptr; cudaGraphExec_t gexec = nullptr;
    CK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
    for (int i = 0; i < iters; ++i) once();
    CK(cudaStreamEndCapture(h->stream, &graph));
    CK(cudaGraphInstantiate(&gexec, graph, 0));
    CK(cudaGraphLaunch(gexec, h->stream));           // warm
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaEventRecord(e0, h->stream));
    CK(cudaGraphLaunch(gexec, h->stream));
    CK(cudaEventRecord(e1, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    cudaGraphExecDestroy(gexec); cudaGraphDestroy(graph);
    if (is_tc && getenv("VTTS_TC_STAMPS")) {
      unsigned long long* d = nullptr;
      CK(cudaMalloc(&d, 16 * 8)); CK(cudaMemset(d, 0, 16 * 8));
      h->tc_dbg = d;
      cudaEvent_t a0, a1; CK(cudaEventCreate(&a0)); CK(cudaEventCreate(&a1));
      CK(cudaEventRecord(a0, h->stream));
      once();
      CK(cudaEventRecord(a1, h->stream));
      CK(cudaStreamSynchronize(h->stream));
      h->tc_dbg = nullptr;
      unsigned long long st[16];
      CK(cudaMemcpy(st, d, sizeof(st), cudaMemcpyDeviceToHost));
      float one = 0.f; CK(cudaEventElapsedTime(&one, a0, a1));
      fprintf(stderr, "[tc stamps %s] event %.2f us | entry->setup %.2f | ->first TMA issued %.2f | ->all TMA issued %.2f | ->first full %.2f | ->mma issued %.2f | ->acc ready %.2f | ->epi done %.2f | ->sync %.2f (us since entry)\n",
              what, one * 1e3, (st[1] - st[0]) / 1e3, (st[2] - st[0]) / 1e3, (st[3] - st[0]) / 1e3, (st[4] - st[0]) / 1e3,
              (st[5] - st[0]) / 1e3, (st[6] - st[0]) / 1e3, (st[7] - st[0]) / 1e3, (st[8] - st[0]) / 1e3);
      cudaFree(d); cudaEventDestroy(a0); cudaEventDestroy(a1);
    }
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    result = ms / iters;
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    h->profiling = prof0;
    for (void* p2 : {(void*)dl, (void*)dof, (void*)x, (void*)y, (void*)w, (void*)bias, (void*)ph, (void*)pl, (void*)wh, (void*)wl}) if (p2) cudaFree(p2);
    h->B = B0; h->h_frm_len = fl0; h->h_tok_len = tl0; h->v_frm_len = vf0; h->v_tok_len = vt0;
  });
  return rc == VTTS_OK ? result : (float)rc;
}

}  // extern "C"
