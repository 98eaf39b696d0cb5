"""Where the batch-1 flow's and decoder's time goes, for the bench utterance (bench.workload: 128 phonemes, precision mode 1).

Prints, from one process on one GPU:
  1. the in-graph entry-to-entry time of each of the flow's 68 launches (17 per coupling layer: pre, qkv, attn, o, ln1, ffn1,
     ffn2, ln2, in_i / rs_i per WN layer, post) and of the decoder's 19 (vtts_timeline stamps, %globaltimer), with the split
     plan of every tensor-core launch (conv launch log) and its MMA and L2-byte floors computed from that plan;
  2. the TC_STAMP intervals of CTA 0 for the flow's two dominant tensor-core shapes (the WN in-conv, k = 5; a 1x1 conv), one
     launch of each MRF stage, the stage-2 upsampling and conv_post, each run alone through Engine.microbench
     (VTTS_TC_STAMPS), with the column pairs each epilogue thread finishes under that launch's plan;
  3. the GPU's name, power limit and SM clocks, read in the same run.

The microbench runs one problem per launch, so its MRF launches are the largest resblock (k = 11) alone, not the grouped
k = 11 / 7 / 3 launch of the chain, and it launches cold (no predecessor to overlap).  Its split plan is printed beside it.
Its epilogue is bias + fp32 rows, one residual-free store pair per column pair.
Floors: MMA = the longest CTA's k-steps x 3 bf16 MMAs of 128 x BN x 64 at one SM's share of the data-sheet 989 TFLOP/s
(dense bf16, 700 W); L2 bytes = every k-step's activation (2 planes x 128 rows x 128 B) and weight (2 planes x BN x 128 B)
tiles over an assumed L2 -> SM rate (L2_TBS, default 5.5 TB/s; not measured here).
usage: python tools/decoder_phases.py [out.json]"""
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vosk_tts_b200 import config as C, synthetic, weights  # noqa: E402
from vosk_tts_b200.engine import Engine  # noqa: E402
import bench  # noqa: E402

PEAK_BF16 = 989e12          # dense bf16, H100 SXM data sheet (700 W)
N_SM = 132
L2_TBS = float(os.environ.get("L2_TBS", "5.5"))
TC_BM, TC_BK = 128, 64


def stamp_names():
    """source line of each PDL_LAUNCH -> kernel name (the headers that stamp share the line space of the timeline)"""
    names = {}
    for fn in ("kernels.cuh", "conv_tc.cuh", "attn_tc.cuh"):
        cur = None
        for i, line in enumerate(open(os.path.join(ROOT, "vosk_tts_b200", "csrc", fn)), 1):
            m = re.search(r"^(?:__global__.*?\s|__device__.*?\s|)(\w+_kernel|conv_tc_body)\s*\(", line)
            if m:
                cur = m.group(1)
            if "PDL_LAUNCH();" in line and cur:
                names[i] = "conv_tc" if cur == "conv_tc_body" else cur
    return names


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def decoder_problems(cfg, frames):
    """(label, [(Cin, Cout, k, rows)] per problem) of the decoder's 16 tensor-core launches, in launch order"""
    ch, rm = cfg["upsample_initial_channel"], 1
    out = [("conv_pre", [(cfg["inter_channels"], ch, 7, frames)])]
    nk = len(cfg["resblock_kernel_sizes"])
    for i, u in enumerate(cfg["upsample_rates"]):
        kp = cfg["upsample_kernel_sizes"][i] // u
        out.append(("ups%d" % i, [(ch, ch // 2, kp, frames * rm)] * u))
        rm *= u
        ch //= 2
        for d in range(len(cfg["resblock_dilation_sizes"][0])):
            for half in ("c1", "c2"):
                ks = list(reversed(cfg["resblock_kernel_sizes"]))      # heaviest resblock first (mrf_heavy_first)
                out.append(("mrf%d.d%d.%s" % (i, d, half), [(ch, ch, k, frames * rm) for k in ks[:nk]]))
    pc = cfg["subbands"] * (cfg["gen_istft_n_fft"] + 2)
    out.append(("conv_post", [(ch, pc, 7, frames * rm + 1)]))
    return out


def flow_problems(cfg, frames):
    """(role, [(Cin, Cout, k, rows)] per problem, or None for a launch that is not a tensor-core conv) of one coupling layer's
    17 launches, in launch order (engine.cu flow_tc / wn_tc; transformer flows)"""
    H, half, fk, nl = cfg["hidden_channels"], cfg["inter_channels"] // 2, cfg["flow_kernel_size"], cfg["flow_wn_layers"]
    out = [("pre", None), ("qkv", [(H, 3 * H, 1, frames)]), ("attn", None), ("o", [(H, H, 1, frames)]), ("ln1", None),
           ("ffn1", [(H, H, fk, frames)]), ("ffn2", [(H, H, fk, frames)]), ("ln2", None)]
    for i in range(nl):
        out.append(("in%d" % i, [(H, 2 * H, fk, frames)]))
        out.append(("rs%d" % i, [(H, H, 1, frames)] * (2 if i < nl - 1 else 1)))
    out.append(("post", [(H, half, 1, frames)]))
    return out


def epi_pairs(rep):
    """column pairs each consumer thread finishes in the epilogue of a one-problem launch: (BN / split) / 4"""
    return rep["bn"] // max(rep["split"], 1) // 4


def floors(probs, rep):
    """MMA and L2-byte floors (us) of one launch from its plan (bn, psplit)"""
    bn = rep["bn"]
    flop_step = 3 * 2.0 * TC_BM * bn * TC_BK
    a_step, w_step = 2 * TC_BM * 128, 2 * bn * 128
    crit, nbytes = 0, 0.0
    for p, (cin, cout, k, rows) in enumerate(probs):
        s = rep["psplit"][p] if rep["split"] > 1 else 1
        steps = cin // TC_BK * k
        tiles = -(-rows // TC_BM) * -(-cout // bn)
        crit = max(crit, -(-steps // max(s, 1)))
        nbytes += tiles * steps * (a_step + w_step)
    return dict(crit_steps=crit, mma_us=crit * flop_step / (PEAK_BF16 / N_SM) * 1e6, l2_mb=nbytes / 1e6,
                l2_us=nbytes / (L2_TBS * 1e12) * 1e6)


def plan_str(rep):
    return "bn%d split%d psplit%s grid(%d,%d,%d)" % (rep["bn"], rep["split"], rep["psplit"][:4], rep["grid_x"], rep["grid_y"],
                                                    rep["grid_z"])


def stamps(eng, spec):
    """TC_STAMP intervals of CTA 0 for one cold microbench launch of `spec` (the kernel prints them to stderr)"""
    os.environ["VTTS_TC_STAMPS"] = "1"
    with tempfile.TemporaryFile(mode="w+") as f:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            eng.conv_log(1)
            us = eng.microbench(spec, 20) * 1e3
            log = eng.conv_log(2)
            eng.conv_log(0)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        txt = f.read()
    del os.environ["VTTS_TC_STAMPS"]
    m = re.search(r"event ([\d.]+) us \| entry->setup ([\d.]+) \| ->first TMA issued ([\d.]+) \| ->all TMA issued ([\d.]+) \| "
                  r"->first full ([\d.]+) \| ->mma issued ([\d.]+) \| ->acc ready ([\d.-]+) \| ->epi done ([\d.]+) \| ->sync ([\d.]+)", txt)
    if not m:
        raise SystemExit("no stamp line from microbench %s:\n%s" % (spec, txt))
    ev, s1, s2, s3, s4, s5, _s6, s7, s8 = (float(v) for v in m.groups())
    iv = {"launch->entry (event - CTA0 entry->exit)": ev - s8, "entry->wait": s1, "wait->first full": s4 - s1,
          "k-loop (first full->end)": s5 - s4, "reduce+epilogue": s7 - s5, "exit barriers": s8 - s7,
          "producer: first issue->last issue": s3 - s2}
    return dict(spec=spec, graph_us_per_launch=us, event_us=ev, plan=plan_str(log[-1]), pairs=epi_pairs(log[-1]), intervals=iv,
                rep=log[-1])


def main():
    cfg = C.DEFAULT_CONFIG
    wl = bench.workload(cfg)
    info = gpu_info()
    blob, man = weights.pack(weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 1234)), cfg)
    eng = Engine(cfg, blob, man, device=0, precision=1)
    run = lambda: eng.infer(wl["tok"], wl["lens"], wl["sid"], wl["scales"], wl["eps_dp"],  # noqa: E731
                            lambda mf: wl["eps_z"][:, :, :mf])
    ylen = eng.durations(wl["tok"], wl["lens"], wl["sid"], wl["scales"], wl["eps_dp"])
    frames = int(np.asarray(ylen[0] if isinstance(ylen, tuple) else ylen).reshape(-1)[0])
    eng.conv_log(1)
    run()                                  # captures the graphs: the host enqueues every launch once
    log = eng.conv_log(2)
    eng.conv_log(0)
    for _ in range(4):
        run()
    eng.timeline(1)
    run()
    tl = eng.timeline(2)
    eng.timeline(0)
    tl = tl[np.argsort(tl[:, 1])]
    names = stamp_names()
    # (negative lines are phase stamps inside a kernel, not launch entries)
    seq = [(names.get(int(ln), "line%d" % int(ln)), int(t)) for ln, t in tl if int(ln) < 1 << 63]
    means = [i for i, (n, _) in enumerate(seq) if n == "mrf_mean_planes_kernel"]
    if len(means) < 2:
        raise SystemExit("decoder not found in the timeline: %s" % [n for n, _ in seq])
    m2 = means[-1]
    s0 = m2 - 16
    dec = seq[s0:m2 + 3]
    expect = ["conv_tc"] * 8 + ["mrf_mean_planes_kernel"] + ["conv_tc"] * 7 + ["mrf_mean_planes_kernel", "conv_tc", "istft_pqmf_kernel"]
    if [n for n, _ in dec] != expect:
        print("warning: unexpected decoder launch sequence, labels below may be off: %s" % [n for n, _ in dec])
    tc_log = [r for r in log if r["use_tc"]]
    probs = decoder_problems(cfg, frames)
    dec_reps = tc_log[-len(probs):]
    rows = []
    tci = 0
    for i, (n, t) in enumerate(dec):
        nxt = seq[s0 + i + 1][1] if s0 + i + 1 < len(seq) else None
        r = {"kernel": n, "entry_to_next_us": None if nxt is None else (nxt - t) / 1e3}
        if n == "conv_tc":
            label, pr = probs[tci]
            rep = dec_reps[tci]
            r.update(label=label, plan=plan_str(rep), **floors(pr, rep))
            tci += 1
        else:
            r["label"] = n.replace("_kernel", "")
        rows.append(r)
    total = (dec[-1][1] - dec[0][1]) / 1e3 + (rows[-1]["entry_to_next_us"] or 0.0)
    # the flow: the coupling layers' launches right before the decoder's conv_pre (the flow's post conv writes the planes
    # conv_pre reads, so no split_planes launch lies between them)
    layer = flow_problems(cfg, frames)
    nfl = cfg["flow_n_flows"] * len(layer)
    f0 = s0 - nfl
    flow = seq[f0:s0]
    fexpect = [("conv_tc" if pr else None) for _, pr in layer] * cfg["flow_n_flows"]
    if f0 < 0 or any((n == "conv_tc") != (e == "conv_tc") for (n, _), e in zip(flow, fexpect)):
        print("warning: unexpected flow launch sequence, labels below may be off: %s" % [n for n, _ in flow])
    ntc = sum(1 for _, pr in layer if pr) * cfg["flow_n_flows"]
    flow_reps = tc_log[-len(probs) - ntc:-len(probs)]
    frows = []
    tci = 0
    for i, (n, t) in enumerate(flow):
        role, pr = layer[i % len(layer)]
        r = {"label": "f%d.%s" % (i // len(layer), role), "role": role, "kernel": n, "entry_to_next_us": (seq[f0 + i + 1][1] - t) / 1e3}
        if pr and n == "conv_tc":
            rep = flow_reps[tci]
            r.update(plan=plan_str(rep), pairs=epi_pairs(rep) if len(pr) == 1 else None, **floors(pr, rep))
            tci += 1
        frows.append(r)
    flow_total = (dec[0][1] - flow[0][1]) / 1e3
    specs = {"flow WN in (k=5)": "tc:%d:%d:5:1:%d" % (cfg["hidden_channels"], 2 * cfg["hidden_channels"], frames),
             "flow 1x1": "tc:%d:%d:1:1:%d" % (cfg["hidden_channels"], cfg["hidden_channels"], frames),
             "mrf stage 1 (k=11 alone)": "tc:%d:%d:11:1:%d" % (256, 256, frames * 4),
             "mrf stage 2 (k=11 alone)": "tc:%d:%d:11:1:%d" % (128, 128, frames * 16),
             "ups1 (one phase alone)": "tc:%d:%d:4:1:%d" % (256, 128, frames * 4),
             "conv_post": "tc:%d:%d:7:1:%d" % (128, 72, frames * 16 + 1)}
    st = {k: stamps(eng, v) for k, v in specs.items()}
    eng.close()

    print("GPU: %s" % json.dumps(info))
    print("utterance: %d frames, flow in-graph time (first pre conv entry -> decoder conv_pre entry): %.1f us" % (frames, flow_total))
    print("%-3s %-16s %-20s %9s  %-44s %6s %5s %8s %8s %8s" % ("#", "launch", "kernel", "in-graph", "plan", "steps", "pairs",
                                                              "mma_us", "l2_MB", "l2_us"))
    for i, r in enumerate(frows):
        if "plan" in r:
            print("%-3d %-16s %-20s %9.2f  %-44s %6d %5s %8.2f %8.1f %8.2f" % (
                i, r["label"], r["kernel"], r["entry_to_next_us"], r["plan"], r["crit_steps"], r["pairs"] or "-", r["mma_us"],
                r["l2_mb"], r["l2_us"]))
        else:
            print("%-3d %-16s %-20s %9.2f" % (i, r["label"], r["kernel"], r["entry_to_next_us"]))
    print("flow time per role, summed over the coupling layers (us):")
    print("  " + "  ".join("%s %.1f" % (role, sum(r["entry_to_next_us"] for r in frows if r["role"] == role)) for role, _ in layer))
    ftc = [r["entry_to_next_us"] for r in frows if "plan" in r]
    print("flow tensor-core launches: %d, sum %.1f us, mean %.2f us; other flow launches: %.1f us" % (
        len(ftc), sum(ftc), sum(ftc) / max(len(ftc), 1), flow_total - sum(ftc)))
    print("decoder in-graph time (conv_pre entry -> end of the iSTFT tail's interval): %.1f us" % total)
    print("%-3s %-16s %-20s %9s  %-44s %6s %8s %8s %8s" % ("#", "launch", "kernel", "in-graph", "plan", "steps", "mma_us", "l2_MB",
                                                         "l2_us"))
    for i, r in enumerate(rows):
        e = "%9.2f" % r["entry_to_next_us"] if r["entry_to_next_us"] is not None else "      n/a"
        if "plan" in r:
            print("%-3d %-16s %-20s %s  %-44s %6d %8.2f %8.1f %8.2f" % (i, r["label"], r["kernel"], e, r["plan"], r["crit_steps"], r["mma_us"],
                                                                     r["l2_mb"], r["l2_us"]))
        else:
            print("%-3d %-16s %-20s %s" % (i, r["label"], r["kernel"], e))
    mrf = [r["entry_to_next_us"] for r in rows if r["label"].startswith("mrf") and r["kernel"] == "conv_tc"]
    print("MRF launches: %d, sum %.1f us, mean %.2f us; other decoder launches: %.1f us" % (len(mrf), sum(mrf), sum(mrf) / len(mrf),
                                                                                        total - sum(mrf)))
    print("CTA 0 stamp intervals (us), one cold launch each through Engine.microbench:")
    for k, v in st.items():
        print("  %-26s %-22s event %.2f us, in-graph back-to-back %.2f us/launch, plan %s, %d pairs/thread" % (
            k, v["spec"], v["event_us"], v["graph_us_per_launch"], v["plan"], v["pairs"]))
        print("    " + "  ".join("%s %.2f" % kv for kv in v["intervals"].items()))
    if len(sys.argv) > 1:
        json.dump(dict(gpu=info, frames=frames, flow_us=flow_total, flow_launches=frows, decoder_us=total, launches=rows,
                       stamps={k: {kk: vv for kk, vv in v.items() if kk != "rep"} for k, v in st.items()}),
                  open(sys.argv[1], "w"), indent=1)


if __name__ == "__main__":
    main()
