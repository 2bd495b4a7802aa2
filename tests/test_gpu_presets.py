"""`-m gpu`: the weight-stream programs (sampler `samp:`, LM stack `lmf:`, codec `decf:` / `encb:`) at the real widths of every preset and
at every batch size the engine accepts, against the CPU oracle.

At 1.5B / 7B widths and B >= 5 the programs hold 10..16 LM rows (MMA height 32) and the codec's T = 4 stages 32 rows (height 64); at 7B
the gate/up and down projections and, at B = 8, the attention merge of the o-projection then need more shared memory for their
activation operand than the weight ring leaves, and run as K slices.  Tolerances as in test_gpu_parity.py: 2e-4 sampler latents,
2e-3 codec frames and LM hidden states (bf16 KV cache).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from vibevoice_b200.configuration import preset_config
from vibevoice_b200.synth import SynthTokenizer, synth_state_dict

from test_gpu_parity import SEED, _lm_roundtrip, _run_sampler, rel_l2, report
from test_gpu_scale import PARTS, _structured_kv

_STATE = {}


def _state(preset):
    """One synthetic state dict per preset (bf16, what the engine loads); the two most recent presets are kept."""
    if preset not in _STATE:
        while len(_STATE) >= 2:
            _STATE.pop(next(iter(_STATE)))
        cfg = preset_config(preset)
        _STATE[preset] = {"cfg": cfg, "sd": synth_state_dict(cfg, SEED, torch.bfloat16, parts=PARTS)}
    return _STATE[preset]


def _oracle_weights(preset):
    """fp32 copy of the state dict: the oracle up-casts every weight it touches on every call, which at 7B widths would dominate the run."""
    st = _state(preset)
    if "sdf" not in st:
        st["sdf"] = {k: (v.float() if torch.is_tensor(v) and v.dtype == torch.bfloat16 else v) for k, v in st["sd"].items()}
    return st["sdf"]


def _model(preset, B, oracle=True):
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    st = _state(preset)
    cfg = st["cfg"]
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=B)
    m.load_state_dict(st["sd"], tok)
    return m, cfg, tok, (_oracle_weights(preset) if oracle else None)


# ---- sampler -------------------------------------------------------------------------------------------------------------------------
def _sampler_checks(model, cfg, sdf, B, tag, steps_list=(10, 30), sde=False, ragged=True):
    from oracle import vv_oracle as O
    H = cfg.decoder_config.hidden_size
    g = torch.Generator().manual_seed(B * 101 + H)
    for steps in steps_list:
        pos, neg = torch.randn(B, H, generator=g), torch.randn(B, H, generator=g)
        noise = torch.randn(2 * B, 64, generator=g)
        got = _run_sampler(model, cfg, None, pos, neg, noise[:B], list(range(B)), 1.3, steps)
        want = O.sample_speech_tokens(sdf, pos, neg, 1.3, steps, noise)
        e = rel_l2(got, want)
        report("sampler_presets", preset=tag, B=B, steps=steps, rel_l2=e)
        assert e < 2e-4, (tag, B, steps, e)
    if ragged:
        rows = [r for r in range(B) if r % 3 != 1] or [0]        # every row of a 1-prompt batch; otherwise holes in the batch
        n = len(rows)
        pos, neg = torch.randn(n, H, generator=g), torch.randn(n, H, generator=g)
        nz = torch.randn(n, 64, generator=g)
        got = _run_sampler(model, cfg, None, pos, neg, nz, rows, 1.5, 10)
        want = O.sample_speech_tokens(sdf, pos, neg, 1.5, 10, torch.cat([nz, nz]))
        e = rel_l2(got, want)
        report("sampler_presets_ragged", preset=tag, B=B, rows=rows, rel_l2=e)
        assert e < 2e-4, (tag, B, rows, e)
    if sde:
        eng = model.engine
        eng.set_scheduler(eng.scheduler.from_config(eng.scheduler.config, algorithm_type="sde-dpmsolver++", beta_schedule="squaredcos_cap_v2"))
        steps = 10
        pos, neg = torch.randn(B, H, generator=g), torch.randn(B, H, generator=g)
        noise = torch.randn(2 * B, 64, generator=g)
        step_noise = [torch.randn(2 * B, 64, generator=g) for _ in range(steps)]
        eng.set_diffusion_steps(steps)
        eng.upload_step_noise(lambda i: step_noise[i], list(range(B)))
        got = _run_sampler(model, cfg, None, pos, neg, noise[:B], list(range(B)), 1.3, steps)
        want = O.sample_speech_tokens(sdf, pos, neg, 1.3, steps, noise, algorithm_type="sde-dpmsolver++", step_noise=step_noise)
        ode = O.sample_speech_tokens(sdf, pos, neg, 1.3, steps, noise)
        e = rel_l2(got, want)
        report("sampler_presets_sde", preset=tag, B=B, rel_l2=e, moved_from_ode=rel_l2(want, ode))
        assert e < 2e-4 and rel_l2(want, ode) > 100 * e, (tag, B, e)


@pytest.mark.parametrize("B", [1, 4, 5, 8])
@pytest.mark.parametrize("preset", ["1.5b-l2", "7b-l2"])
def test_sampler_vs_oracle_at_real_widths(preset, B):
    """The 10- and 30-step (301-stage) sampler programs, a ragged active set, and at B = 5 the SDE solver with injected step noise."""
    model, cfg, tok, sdf = _model(preset, B)
    try:
        _sampler_checks(model, cfg, sdf, B, preset, sde=(B == 5))
    finally:
        model.engine.close()


# ---- codec ---------------------------------------------------------------------------------------------------------------------------
def _codec_checks(model, cfg, sdf, B, tag, n_frames=12):
    """Decoder + semantic encoder frame by frame with ragged active sets and a <speech_end> state zeroing in the middle: after 12 frames the
    k = 7 mixer histories and the conv histories hold real frames."""
    from oracle import vv_oracle as O
    eng = model.engine
    eng.codec_state_reset()
    a, s = O.StreamState(B), O.StreamState(B)
    g = torch.Generator().manual_seed(50 + B)
    scale, bias = float(sdf["model.speech_scaling_factor"]), float(sdf["model.speech_bias_factor"])
    worst_a = worst_s = 0.0
    for f in range(n_frames):
        rows = list(range(B)) if f % 3 != 2 or B == 1 else [r for r in range(B) if (r + f) % 2 == 0]
        if f == n_frames // 2:
            zr = [0] if B == 1 else [0, B - 1]
            eng.codec_state_zero(zr); a.set_to_zero(zr); s.set_to_zero(zr)
        lat = torch.randn(len(rows), 64, generator=g)
        full = torch.zeros(B, 64)
        full[rows] = lat
        with torch.cuda.stream(eng.stream):
            eng.latent.copy_(full.cuda())
        eng.upload_frame_inputs(torch.zeros(len(rows), 64), rows)
        eng.codec_decode()
        eng.semantic_encode()
        eng.sync()
        audio = O.decoder_frame(sdf, cfg.acoustic_tokenizer_config, (lat / scale - bias)[:, None, :], a, rows)
        sem = O.encoder_frame(sdf, cfg.semantic_tokenizer_config, audio, s, rows)
        ea = rel_l2(eng.audio.cpu()[rows], audio[:, 0])
        es = rel_l2(eng.feat.cpu()[rows], sem[:, 0])
        worst_a, worst_s = max(worst_a, ea), max(worst_s, es)
        report("codec_presets", preset=tag, B=B, frame=f, rows=rows, audio_rel_l2=ea, sem_rel_l2=es)
        assert ea < 2e-3 and es < 2e-3, (tag, B, f, rows, ea, es)
    return worst_a, worst_s


@pytest.mark.parametrize("B", [1, 4, 8])
def test_streaming_codec_vs_oracle_at_real_widths(B):
    """The 1.5B codec widths (the same for 7B): C up to 2048; at B = 8 the T = 4 stages run 32 rows (MMA height 64)."""
    model, cfg, tok, sdf = _model("1.5b-l2", B)
    try:
        _codec_checks(model, cfg, sdf, B, "1.5b-l2")
    finally:
        model.engine.close()


# ---- LM decode -----------------------------------------------------------------------------------------------------------------------
def _lm_checks(model, cfg, sdf, B, tag, pos_len, neg_len, n_steps=4):
    """Positive rows at `pos_len` tokens, negative rows at `neg_len` (structured bf16 prefixes imported through vv_kv_write), n_steps
    decode steps with the negative rows advancing every other step, against qwen2_forward over the same prefixes."""
    from oracle import vv_oracle as O
    eng = model.engine
    dc = cfg.decoder_config
    nl, nkv, hd = dc.num_hidden_layers, dc.num_key_value_heads, dc.head_dim
    lens = list(pos_len) + list(neg_len)
    assert len(lens) == 2 * B
    eng.kv_init(sum(lens) + 2 * B * (n_steps + 64))
    g = torch.Generator().manual_seed(sum(lens))
    caches = [O.KVCache(nl, kv_bf16=True) for _ in range(2 * B)]
    for seq, L in enumerate(lens):
        eng.kv_set_len(seq, 0)
        if L == 0:
            continue
        for layer in range(nl):
            k, v = _structured_kv(nkv, L, hd, g)
            caches[seq].preload(layer, k.float(), v.float())
            kd, vd = k.transpose(0, 1).contiguous().cuda(), v.transpose(0, 1).contiguous().cuda()
            with torch.cuda.stream(eng.stream):
                eng.kv_write(seq, layer, 0, kd, vd)
            eng.sync()
        eng.kv_set_len(seq, L)
    errs = []
    for step in range(n_steps):
        x = torch.randn(2 * B, dc.hidden_size, generator=g) * 0.05
        with torch.cuda.stream(eng.stream):
            eng.embeds.copy_(x.cuda())
        eng.lm_decode()
        eng.read_tokens()
        adv = [1] * B + [step % 2] * B
        want = []
        for r in range(2 * B):
            n0 = len(caches[r])
            want.append(O.qwen2_forward(sdf, dc, x[r][None], caches[r], n0)[0])
            if not adv[r]:
                caches[r].truncate(n0)
        eng.kv_commit(adv)
        got = eng.hidden.cpu()
        errs.append([rel_l2(got[r], want[r]) for r in range(2 * B)])
    report("lm_decode_presets", preset=tag, B=B, pos_len=list(pos_len), neg_len=list(neg_len), rel_l2=errs)
    assert max(max(e) for e in errs) < 2e-3, errs
    for r in range(2 * B):
        assert eng.kv_len(r) == lens[r] + (n_steps if r < B else n_steps // 2)
    return errs


LM_CASES = {  # (positive lengths, negative lengths): one positive row above 30 K, short negative rows, one on each side of a page edge
    ("7b-l2", 4): ([30777, 2500, 4100, 6000], [63, 64, 65, 7]),
    ("7b-l2", 8): ([30777, 2500, 4100, 6000, 3333, 5120, 2049, 4500], [63, 64, 65, 7, 0, 130, 20, 1]),
    ("1.5b-l2", 8): ([31234, 2600, 4097, 5000, 3001, 6144, 2222, 4444], [63, 64, 65, 9, 0, 128, 33, 2]),
}


@pytest.mark.parametrize("preset,B", list(LM_CASES))
def test_lm_decode_vs_oracle_batched_long_context(preset, B):
    model, cfg, tok, sdf = _model(preset, B)
    try:
        pos_len, neg_len = LM_CASES[(preset, B)]
        _lm_checks(model, cfg, sdf, B, preset, pos_len, neg_len)
    finally:
        model.engine.close()


# ---- every preset at every batch size --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", list(range(1, 9)))
@pytest.mark.parametrize("preset", ["tiny", "tiny64", "1.5b-l2", "7b-l2", "streaming-0.5b-l4"])
def test_every_preset_runs_at_every_batch_size(preset, B):
    """vv_create accepts max_batch 1..8 for every model: one LM decode, one sampler call and one codec frame must succeed and stay finite."""
    model, cfg, tok, _ = _model(preset, B, oracle=False)
    try:
        eng = model.engine
        g = torch.Generator().manual_seed(B)
        H = cfg.decoder_config.hidden_size
        eng.kv_init(512)
        for seq in range(2 * B):
            eng.kv_set_len(seq, 0)
        with torch.cuda.stream(eng.stream):
            eng.embeds.copy_((torch.randn(2 * B, H, generator=g) * 0.05).cuda())
        eng.lm_decode()
        eng.read_tokens()
        eng.set_diffusion_steps(10)
        eng.upload_frame_inputs(torch.randn(B, 64, generator=g), list(range(B)))
        eng.diffusion_sample(1.3)
        eng.codec_decode()
        eng.semantic_encode()
        eng.sync()
        for name in ("hidden", "logits", "latent", "audio", "feat"):
            t = getattr(eng, name)
            assert torch.isfinite(t).all(), (preset, B, name)
        assert eng.latent.abs().sum() > 0 and eng.audio.abs().sum() > 0
    finally:
        model.engine.close()


# ---- the fallback instantiations ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("switch", ["VV_STREAM_GENERIC", "VV_STREAM_NO_NB16"])
def test_program_families_on_fallback_kernels(monkeypatch, switch):
    """Every program family once more on the all-features kernel (VV_STREAM_GENERIC=1; otherwise picked only for programs no specialised
    variant covers) and without the compile-time 16-row operand (VV_STREAM_NO_NB16=1).  Both are read when a program is built, i.e. on
    the first call of each family of a fresh engine."""
    monkeypatch.setenv(switch, "1")
    model, cfg, tok, sdf = _model("1.5b-l2", 2)
    try:
        _sampler_checks(model, cfg, sdf, 2, "1.5b-l2 " + switch, steps_list=(10,), ragged=False)
        _codec_checks(model, cfg, sdf, 2, "1.5b-l2 " + switch, n_frames=4)
        errs = _lm_roundtrip(model, cfg, tok, sdf, n_prompt=20, n_steps=4)
        report("lm_decode_fallback_kernels", switch=switch, max_rel_l2=max(errs))
        assert max(errs) < 2e-3, errs
    finally:
        model.engine.close()
