"""A/B of the launch shapes of two builds of libvtts.so: every entry point of every model family (seeded synthetic weights), at
B = 1 and on a ragged batch, in precision modes 0, 1 and 2.  One process per library (VTTS_LIB) prints, per call, the
conv-launch log, the launch counts and a SHA-256 of every output; the two transcripts must be equal line for line.  Two
passes: graphs off with the profiler on (its FLOPs too), then graphs on with the profiler off (which bypasses graphs), each
call made twice so that the second replays the graph the first captured.
usage: python tools/ab_launch.py libA.so libB.so [out_dir]"""
import difflib
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r'''
import hashlib, json, os, sys
ROOT = sys.argv[1]
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from vosk_tts_b200 import config as C, synthetic, weights
from vosk_tts_b200.engine import Engine
from vosk_tts_b200.stabletts import StableTTS
import bert_inputs as BI, contentvec_inputs as CI, hifigan_inputs as HI, quickvc_convert_inputs as QC, quickvc_inputs as QI
import stabletts_cfm_inputs as SI, stabletts_inputs as TI, t2s_inputs as T2
from vosk_tts_b200.gpt_sovits import Text2Semantic

GRAPHED = False                            # the pass: graphs off and the profiler on, or graphs on and the profiler off


def digest(x):
    if isinstance(x, dict):
        return {k: digest(v) for k, v in sorted(x.items())}
    if isinstance(x, (list, tuple)):
        return [digest(v) for v in x]
    if isinstance(x, np.ndarray) or np.isscalar(x):
        a = np.ascontiguousarray(x)
        return "%s%s:%s" % (a.dtype, list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()[:24])
    return repr(x)


def run(eng, name, fn):
    eng.conv_log(1)
    eng.profile(not GRAPHED)
    try:
        out = digest([fn(), fn()] if GRAPHED else fn())
    except Exception as e:                 # (a refusal is part of the transcript too)
        out = "error: %s" % e
    log = eng.conv_log(2)
    eng.conv_log(0)
    rec = {"call": name, "out": out, "kernel_launches": eng.kernel_launches()}
    if not GRAPHED:
        p = eng.profile_read()
        rec.update(conv_launches=p["conv_launches"], conv_flops=p["conv_flops"], tc_launches=p["tc_launches"], tc_flops=p["tc_flops"])
    print(json.dumps(rec))
    for r in log:
        print("  " + json.dumps(r, sort_keys=True))
    sys.stdout.flush()


def engine(cfg, blob, man, p):
    e = Engine(cfg, blob, man, device=0, precision=p)
    e.set_graphs(GRAPHED)
    return e


rng = np.random.RandomState(7)
cfg = C.DEFAULT_CONFIG
vblob, vman = weights.pack(weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 1234, posterior=True)), cfg, posterior=True)
qcfg = QI.config()
sblob, sman = weights.pack_quickvc(weights.fold_weight_norm(QI.speaker_encoder()), qcfg)
ccfg = dict(qcfg, contentvec=CI.cv())
cblob, cman = weights.pack_quickvc(weights.fold_weight_norm(QC.model()), qcfg, contentvec=CI.model())
scfg = SI.config()
fblob, fman = weights.pack_stabletts_cfm(SI.model(scfg), scfg)
tcfg = TI.config()


def vits2(p, batch, tag):
    e = engine(cfg, vblob, vman, p)
    T = [9 * k + 3 for k in batch]
    ids = np.zeros((len(T), max(T)), np.int64)
    for b, t in enumerate(T):
        ids[b, :t] = rng.randint(1, cfg["n_vocab"], t)
    sid = list(range(len(T)))
    sc = (0.667, 1.0, 0.8)
    run(e, tag + " infer", lambda: e.infer(ids, T, sid, sc, seed=1))
    run(e, tag + " durations", lambda: e.durations(ids, T, sid, sc, seed=2, want_durations=True))
    run(e, tag + " synthesize", lambda: e.synthesize(e.durations(ids, T, sid, sc, seed=2)))
    run(e, tag + " synthesize alignment", lambda: e.synthesize(e.durations(ids, T, sid, sc, seed=2), want_alignment=True))
    run(e, tag + " flow+decode_chunk", lambda: list(e.synthesize_stream(ids[:1, :T[0]], 1, sc, chunk_frames=40, seed=3)))
    run(e, tag + " convert", lambda: e.convert(wav(batch), sid, sid[::-1], lengths=wl(batch), seed=4))
    run(e, tag + " align", lambda: e.align(ids, T, sid, wav(batch), wl(batch), seed=5))
    clips = [c[:n] for c, n in zip(wav(batch), wl(batch))]
    for fr, to in ((16000, 22050), (22050, 22050)):
        run(e, tag + " resample %d->%d" % (fr, to), lambda: e.resample(clips, fr, to, trim_top_db=20, return_bounds=True))
    e.close()


def quickvc(p, batch, tag):
    e = engine(qcfg, sblob, sman, p)
    run(e, tag + " speaker_embedding", lambda: e.speaker_embedding(wav(batch), wl(batch)))
    F = [60 * k + 71 for k in batch]
    mel = np.random.RandomState(12).normal(-4.0, 2.0, (len(F), qcfg["n_mel_channels"], max(F))).astype(np.float32)
    run(e, tag + " speaker_embedding_mel", lambda: e.speaker_embedding_mel(mel, F))
    e.close()
    e = engine(ccfg, cblob, cman, p)
    U = [13 * k + 4 for k in batch]
    units = [QC.units(u, 10 + i) for i, u in enumerate(U)]
    g = np.random.RandomState(8).rand(len(U), qcfg["gin_channels"]).astype(np.float32)
    run(e, tag + " quickvc_convert", lambda: e.quickvc_convert(units if len(U) > 1 else units[0], g if len(U) > 1 else g[0], seed=6))
    run(e, tag + " content_units", lambda: e.content_units(wav(batch), wl(batch)))
    run(e, tag + " quickvc_convert_wav", lambda: e.quickvc_convert_wav(wav(batch), g, wl(batch), seed=7))
    e.close()


def stabletts(p, batch, tag):
    e = engine(scfg, fblob, fman, p)
    mus = [SI.inputs("ab", 17 * k + 5, scfg)[0].T for k in batch]
    for s in (0.0, 0.5):
        run(e, tag + " cfm_decode s=%g" % s, lambda: e.cfm_decode(mus if len(mus) > 1 else mus[0], sid=1, n_timesteps=3, guidance_scale=s, seed=8))
    e.close()
    tts = StableTTS({"n_vocab": tcfg["n_vocab"]}, TI.model(tcfg), device=0, precision=p, vocoder=HI.checkpoint())
    e = tts.engine
    e.set_graphs(GRAPHED)
    r = np.random.RandomState(9)
    L = [7 * k + 4 for k in batch]
    xs = [r.randint(0, tcfg["n_vocab"], (tcfg["n_streams"], t)) for t in L]
    berts = [r.randn(tcfg["bert_dim"], t).astype(np.float32) for t in L]
    for w in (False, True):
        run(e, tag + " stabletts_synthesise wav=%d" % w, lambda: tts.synthesise(xs, berts, 0, n_timesteps=3, seed=9, return_wav=w))
    run(e, tag + " stabletts_synthesise prior", lambda: tts.synthesise(xs, berts, 0, n_timesteps=3, seed=9, return_prior=True))
    mels = [m.T for m in HI.case_mels(("ab", [11 * k + 6 for k in batch]))]
    run(e, tag + " hifigan_vocode", lambda: e.hifigan_vocode(mels if len(mels) > 1 else mels[0]))
    tts.close()


def multistream(p, batch, tag):
    bt = BI.tiny()
    mc = {"n_vocab": 120, "bert_dim": bt["cv_hidden"]}
    tts = StableTTS(mc, synthetic.make_random_stabletts(C.stabletts_config(mc), 8642), device=0, precision=p, vocoder=HI.checkpoint(),
                    bert=(BI.model(bt), bt))
    e = tts.engine
    e.set_graphs(GRAPHED)
    r = np.random.default_rng(10)
    sents = [BI.sentence(bt, 5 * k + 3, salt=k) for k in batch]
    run(e, tag + " bert_features", lambda: tts.bert_features(sents))
    T = [6 * k + 2 for k in batch]
    ids = [r.integers(0, 120, (5, t)).astype(np.int64) for t in T]
    rows = [np.sort(r.integers(0, len(s), t)).astype(np.int32) for s, t in zip(sents, T)]
    pause = [np.where(r.random(t) < 0.1, 3.0, 0.0).astype(np.float32) for t in T]
    run(e, tag + " stabletts_synthesise pieces", lambda: tts.synthesise(ids, None, [b % 2 for b in range(len(T))], pause, n_timesteps=3,
                                                                        seed=11, return_wav=True, pieces=sents, bert_rows=rows))
    tts.close()


def t2s(p, batch, tag):
    sd, c = T2.model(T2.SMALL)
    m = Text2Semantic((sd, c), precision=p)
    e = m.engine
    e.set_graphs(GRAPHED)
    phs = [T2.phones(c, 6 * k + 4, 20 + b) for b, k in enumerate(batch)]
    prs = [T2.prompt(c, 3 * k, 30 + b) for b, k in enumerate(batch)]
    berts = [np.random.default_rng(40 + b).standard_normal((len(x), 1024)).astype(np.float32) * 0.3 for b, x in enumerate(phs)]
    run(e, tag + " t2s_decode", lambda: e.t2s_decode(phs, prs, berts, step_cap=40, seeds=12))
    q = np.stack([T2.q_draws(c, 40, 50 + b) for b in range(len(batch))])
    run(e, tag + " t2s_decode q", lambda: e.t2s_decode(phs, None, None, step_cap=40, q=q, logits_steps=8))
    m.close()


def wl(batch):
    return [4000 * k + 1234 for k in batch]


def wav(batch):
    return (np.random.RandomState(len(batch)).rand(len(batch), max(wl(batch))).astype(np.float32) - 0.5) * 0.4


for GRAPHED in (False, True):
    print(json.dumps({"pass": "graphs on, profiler off" if GRAPHED else "graphs off, profiler on"}))
    for p in (0, 1, 2):
        for batch in ((1,), (3, 1, 2)):
            for fam in (vits2, quickvc, stabletts, multistream, t2s):
                tag = "p%d B%d" % (p, len(batch))
                try:
                    fam(p, batch, tag)
                except Exception as ex:            # an engine the family refuses in this mode
                    print(json.dumps({"family": fam.__name__, "tag": tag, "error": str(ex)}))
'''


def main():
    libs = [os.path.abspath(x) for x in sys.argv[1:3]]
    out_dir = sys.argv[3] if len(sys.argv) > 3 else "."
    os.makedirs(out_dir, exist_ok=True)
    texts = []
    for i, lib in enumerate(libs):
        env = dict(os.environ, VTTS_LIB=lib)
        r = subprocess.run([sys.executable, "-c", CHILD, ROOT], env=env, capture_output=True, text=True)
        path = os.path.join(out_dir, "ab_launch_%s.txt" % "AB"[i])
        with open(path, "w") as f:
            f.write(r.stdout + ("\n[exit %d]\n%s" % (r.returncode, r.stderr[-4000:]) if r.returncode else ""))
        texts.append(r.stdout.splitlines())
        print("%s: exit %d, %d calls, %d lines -> %s" % (lib, r.returncode, sum(not l.startswith(" ") for l in texts[-1]), len(texts[-1]), path))
        if r.returncode:
            print(r.stderr[-2000:])
    diff = list(difflib.unified_diff(texts[0], texts[1], "A", "B", lineterm="", n=1))
    print("identical" if not diff else "DIFFERENT (%d diff lines)\n%s" % (len(diff), "\n".join(diff[:80])))
    sys.exit(0 if not diff and texts[0] else 1)


if __name__ == "__main__":
    main()
