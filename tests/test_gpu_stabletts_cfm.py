"""GPU tests of the StableTTS flow-matching decoder (vtts_cfm_decode) against the float64 oracle and the reference's stored
fp32 mel, and of its kernels alone through the vtts_debug_read taps."""
import numpy as np
import pytest
import torch

import stabletts_cfm_inputs as SI
from oracle import stabletts_cfm_oracle as so
from vosk_tts_b200 import weights
from vosk_tts_b200.engine import Engine, VttsError, live_bytes
from vosk_tts_b200.stabletts import StableTTS

pytestmark = pytest.mark.gpu

# max |mel - float64 oracle| on the normalised mel (|mel| up to 10); measured maxima are in DESIGN.md 4.l, the budgets ~4x.
BUDGET = {0: 1.6e-4, 1: 1.6e-4}


@pytest.fixture(scope="module")
def golden():
    return np.load(SI.GOLDEN)


@pytest.fixture(scope="module")
def model():
    cfg = SI.config()
    sd = SI.model(cfg)
    return cfg, sd, weights.pack_stabletts_cfm(sd, cfg)


@pytest.fixture(scope="module", params=[0, 1], ids=["fp32", "mode1"])
def eng(request, model):
    cfg, sd, (blob, man) = model
    e = Engine(cfg, blob, man, device=0, precision=request.param)
    e.precision = request.param
    yield e
    e.close()


@pytest.fixture(scope="module")
def eng0(model):
    cfg, sd, (blob, man) = model
    e = Engine(cfg, blob, man, device=0, precision=0)
    yield e
    e.close()


def run(e, case, **kw):
    name, lens, n, s, temp, sids = case
    ins = SI.case_inputs(case)
    mel, ln = e.cfm_decode([m.T for m, _ in ins], sids, n_timesteps=n, temperature=temp, guidance_scale=s,
                           noise=[z.T for _, z in ins], **kw)
    assert list(ln) == lens
    return [mel[b, :lens[b]].T for b in range(len(lens))]


@pytest.mark.parametrize("case", SI.CASES, ids=lambda c: c[0])
def test_fixture_cases(eng, case, golden, model):
    cfg, sd, _ = model
    name, lens, n, s, temp, sids = case
    out = run(eng, case)
    worst = 0.0
    for b, (mu, nz) in enumerate(SI.case_inputs(case)):
        o64 = so.decode(sd, cfg, mu, sids[b], nz, n, temp, s, torch.float64)
        e64 = float(np.abs(out[b] - o64).max())
        eref = float(np.abs(out[b] - golden["%s.mel%d" % (name, b)]).max())
        worst = max(worst, e64, eref)
        assert e64 < BUDGET[eng.precision] and eref < BUDGET[eng.precision], (name, b, e64, eref)
    print("cfm %s mode %d: max err %.2e" % (name, eng.precision, worst))


def test_alone_equals_batched_and_eager_equals_replay(eng):
    case = SI.CASES[5]
    first = run(eng, case)                      # eager (and the capture behind it)
    r0 = eng.graph_replays()
    again = run(eng, case)
    assert eng.graph_replays() == r0 + 1
    for a, b in zip(first, again):
        assert np.array_equal(a, b)
    name, lens, n, s, temp, sids = case
    for b in range(len(lens)):
        mu, nz = SI.inputs(name + str(b), lens[b])
        mel, _ = eng.cfm_decode(mu.T, sids[b], n_timesteps=n, temperature=temp, guidance_scale=s, noise=nz.T)
        assert np.array_equal(mel[0].T, first[b]), b


def test_denormalise_and_speaker_rows(eng0, model):
    cfg, sd, _ = model
    mu, nz = SI.inputs("dn", 17)
    a, _ = eng0.cfm_decode(mu.T, 1, n_timesteps=2, noise=nz.T)
    d, _ = eng0.cfm_decode(mu.T, 1, n_timesteps=2, noise=nz.T, denormalise=True)
    assert np.allclose(d, so.denormalise(a, sd), atol=1e-5)
    r, _ = eng0.cfm_decode(mu.T, None, n_timesteps=2, noise=nz.T, spk_rows=sd["spk_emb.weight"][1].numpy())
    assert np.array_equal(r, a)


def test_zero_guidance_is_the_conditional_branch(eng0, model):
    """s = 0 runs no unconditional sequence: equal to the oracle's conditional branch, and to a tiny s's first digits."""
    cfg, sd, _ = model
    mu, nz = SI.inputs("g0", 31)
    a, _ = eng0.cfm_decode(mu.T, 0, n_timesteps=3, guidance_scale=0.0, noise=nz.T)
    assert np.abs(a[0].T - so.decode(sd, cfg, mu, 0, nz, 3, 1.0, 0.0)).max() < BUDGET[0]
    b, _ = eng0.cfm_decode(mu.T, 0, n_timesteps=3, guidance_scale=1e-7, noise=nz.T)
    assert np.abs(a - b).max() < 1e-4


def test_one_step_is_one_euler_step_of_the_oracle(eng0, model):
    cfg, sd, _ = model
    mu, nz = SI.inputs("e1", 19)
    mel, _ = eng0.cfm_decode(mu.T, 1, n_timesteps=1, temperature=0.9, guidance_scale=0.5, noise=nz.T)
    dt = torch.float64
    T = 19
    x = torch.as_tensor(nz, dtype=dt) * 0.9
    cs = so.rope_table(T, 48, dt)
    ada = lambda c: [so.ada_rows(sd, cfg, c, l, dt) for l in range(6)]
    vc = so.estimator(sd, cfg, x, so.cond_proj(sd, cfg, torch.as_tensor(mu, dtype=dt), dt), 0.0, ada(sd["spk_emb.weight"][1].double()), cs, dt)
    vu = so.estimator(sd, cfg, x, so.cond_proj(sd, cfg, sd["fake_content"][0].double().repeat(1, T), dt), 0.0,
                      ada(sd["fake_speaker"][0].double()), cs, dt)
    want = x + 1.0 * (vc + 0.5 * (vc - vu))         # t_span = (0, 1): one step of dt = 1
    assert np.abs(mel[0].T - want.numpy()).max() < BUDGET[0]


def test_philox_noise(eng0):
    mu, nz = SI.inputs("ph", 50)
    a, _ = eng0.cfm_decode(mu.T, 0, n_timesteps=2, seed=11)
    b, _ = eng0.cfm_decode(mu.T, 0, n_timesteps=2, seed=11)
    c, _ = eng0.cfm_decode(mu.T, 0, n_timesteps=2, seed=12)
    assert np.array_equal(a, b) and not np.array_equal(a, c) and np.isfinite(a).all()
    d, _ = eng0.cfm_decode(mu.T, 0, n_timesteps=2, noise=nz.T, seed=11)
    e, _ = eng0.cfm_decode(mu.T, 0, n_timesteps=2, noise=nz.T, seed=12)
    assert np.array_equal(d, e)
    # temperature scales the Philox draw: at temperature 0 the start is x = 0 for every seed
    z0, _ = eng0.cfm_decode(mu.T, 0, n_timesteps=2, temperature=0.0, seed=11)
    z1, _ = eng0.cfm_decode(mu.T, 0, n_timesteps=2, temperature=0.0, seed=12)
    assert np.array_equal(z0, z1)


def test_long_utterance(eng, model):
    """3000 frames: the rotary table at large positions, attention over many key tiles."""
    cfg, sd, _ = model
    mu, nz = SI.inputs("long3000", 3000)
    mel, _ = eng.cfm_decode(mu.T, 1, n_timesteps=2, guidance_scale=0.5, noise=nz.T)
    ref = so.decode(sd, cfg, mu, 1, nz, 2, 1.0, 0.5, torch.float64)
    err = float(np.abs(mel[0].T - ref).max())
    print("cfm 3000 frames mode %d: max err %.2e" % (eng.precision, err))
    assert err < BUDGET[eng.precision]


def test_kernels_alone(eng0, model):
    """The conditioning rows, LayerNorm + modulate, the rotary q / k and the Euler update through the debug taps."""
    cfg, sd, _ = model
    H, NC, heads = cfg["hidden_channels"], cfg["noise_channels"], cfg["n_heads"]
    dk = H // heads
    lens = [37, 12]
    name = "taps"
    ins = [SI.inputs(name + str(b), T) for b, T in enumerate(lens)]
    eng0.debug_flags(1)
    try:
        mel, _ = eng0.cfm_decode([m.T for m, _ in ins], [1, 0], n_timesteps=3, temperature=1.0, guidance_scale=0.5,
                                 noise=[z.T for _, z in ins])
        film = eng0.debug_read("st_film").reshape(3, 6, 2 * H)
        ada = eng0.debug_read("st_ada").reshape(4, 6, 6, H)
        xc = eng0.debug_read("st_cond").reshape(-1, NC + H)
        ropet = eng0.debug_read("st_rope").reshape(-1, dk // 4, 2)
        n1 = eng0.debug_read("st_norm1").reshape(-1, H)
        qkv = eng0.debug_read("st_qkv").reshape(-1, 3 * H)
    finally:
        eng0.debug_flags(0)
    off = [0, lens[0] + 8]
    for b in range(2):
        taps = {}
        ref = so.decode(sd, cfg, ins[b][0], [1, 0][b], ins[b][1], 3, 1.0, 0.5, torch.float64, taps)
        rows = slice(off[b], off[b] + lens[b])
        assert np.abs(film - taps["film"].numpy()).max() < 2e-4          # angles of 1000 t in fp32: see DESIGN.md 4.l
        assert np.abs(ada[b] - taps["ada"].numpy()).max() < 2e-5
        assert np.abs(xc[rows, NC:] - taps["cond"].numpy().T).max() < 2e-5
        assert np.abs(xc[rows, :NC] - ref.T).max() < BUDGET[0]           # x after the last Euler update
        assert np.array_equal(xc[rows, :NC], mel[b, :lens[b]])
        assert np.abs(n1[rows] - taps["norm1"].numpy().T).max() < 1e-4
        T = lens[b]
        cos, sin = so.rope_table(T, dk // 2, torch.float64)
        assert np.abs(ropet[:T, :, 0] - cos.numpy()).max() < 1e-7 and np.abs(ropet[:T, :, 1] - sin.numpy()).max() < 1e-7
        for i, n in enumerate("qkv"):
            want = taps[n].numpy().transpose(1, 0, 2).reshape(T, H)      # [heads, T, dk] -> rows [T][heads * dk]
            assert np.abs(qkv[rows, i * H:(i + 1) * H] - want).max() < 2e-4, n
    # the unconditional branch's adaLN rows are the fake speaker's, the same for both utterances
    assert np.array_equal(ada[2], ada[3]) and not np.array_equal(ada[0], ada[2])


def test_rotary_kernel_is_the_reference_arithmetic(eng0):
    """fp32 theta, fp32 product with the position, then cos / sin: equal to the float64 cos / sin of that fp32 angle."""
    mu, nz = SI.inputs("rp", 700)
    eng0.debug_flags(1)
    try:
        eng0.cfm_decode(mu.T, 0, n_timesteps=1, guidance_scale=0.0, noise=nz.T)
        tab = eng0.debug_read("st_rope").reshape(-1, 24, 2)
    finally:
        eng0.debug_flags(0)
    theta = 1.0 / (10000 ** (torch.arange(0, 48, 2).float() / 48))
    ang = (torch.arange(700).float()[:, None] * theta[None, :]).double()
    assert np.abs(tab[:700, :, 0] - ang.cos().numpy()).max() <= 6e-8 and np.abs(tab[:700, :, 1] - ang.sin().numpy()).max() <= 6e-8


def test_argument_checks(eng0, model):
    cfg, sd, _ = model
    mu, nz = SI.inputs("ac", 5)
    for kw, code in (({"n_timesteps": 0}, -1), ({"n_timesteps": 65}, -1), ({"temperature": float("nan")}, -1),
                     ({"guidance_scale": -0.5}, -1), ({"guidance_scale": float("inf")}, -1)):
        with pytest.raises(VttsError) as ei:
            eng0.cfm_decode(mu.T, 0, **kw)
        assert ei.value.code == code, kw
    for sid in (-1, cfg["n_spks"]):
        with pytest.raises(VttsError, match="speaker id out of range"):
            eng0.cfm_decode(mu.T, sid)
    with pytest.raises(VttsError, match="a speaker is required"):
        eng0.cfm_decode(mu.T, None)
    with pytest.raises(VttsError, match="lengths must be in"):
        eng0.cfm_decode(mu.T[None], 0, lengths=[0])
    with pytest.raises(VttsError) as ei:
        eng0.cfm_decode(mu.T, 0, noise=nz.T[:3])
    assert ei.value.code == -4
    with pytest.raises(VttsError, match="serves VITS2 models; the engine holds a StableTTS model"):
        eng0.durations(np.zeros((1, 4), np.int64), [4], [0], (0.6, 1.0, 0.8))
    with pytest.raises(VttsError, match="serves QuickVC models; the engine holds a StableTTS model"):
        eng0.content_units(np.zeros(16000, np.float32))


def test_other_families_refuse_cfm_decode():
    from vosk_tts_b200 import config as C, synthetic
    cfg = C.DEFAULT_CONFIG
    blob, man = weights.pack(weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 1234)), cfg)
    e = Engine(cfg, blob, man, device=0, precision=0)
    try:
        e.cfg = dict(cfg, **SI.config())
        with pytest.raises(VttsError, match="serves StableTTS models; the engine holds a VITS2 model"):
            e.cfm_decode(np.zeros((4, 256), np.float32), 0)
    finally:
        e.close()


def test_front_end_and_engine_lifetime(model):
    cfg, sd, _ = model
    torch.cuda.synchronize()
    before = live_bytes()
    tts = StableTTS(None, sd, device=0, precision=1)
    mu, nz = SI.inputs("short0", 23)
    out = tts.refine([mu, mu[:, :9]], [1, 0], noise=[nz, nz[:, :9]])
    assert [o.shape for o in out] == [(80, 23), (80, 9)]
    one = tts.refine(mu, 1, noise=nz)
    assert np.array_equal(one, out[0])
    assert live_bytes()[0] > before[0]
    tts.close()
    assert live_bytes() == before
