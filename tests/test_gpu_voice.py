"""`-m gpu` tests of the voice-prompt encoder (a-9, `vv_voice_encode`): the non-streaming acoustic tokenizer encoder, sampling and acoustic
connector on the engine, against the fp32 oracle (`oracle/vv_oracle.py`) on bf16-valued synthetic weights, and voice prompts on the
token-by-token (decode-kernel) prefill of `generate()`."""
import ctypes as C
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from vibevoice_b200 import _native as NV
from vibevoice_b200.configuration import preset_config
from vibevoice_b200.synth import SynthTokenizer, synth_state_dict

SEED = 1234
ENC = "model.acoustic_tokenizer.encoder"
OUT = os.environ.get("VV_REPORT_DIR") or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "reports")


def rel_l2(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def report(name, **kv):
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "parity_report.jsonl"), "a") as f:
        f.write(json.dumps(dict(test=name, **kv)) + "\n")


def make_model(preset, max_batch=1, torch_prefill=False, drop=()):
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    cfg = preset_config(preset)
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, SEED, torch.bfloat16)
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=max_batch, torch_prefill=torch_prefill)
    m.load_state_dict({k: v for k, v in sd.items() if not any(k.startswith(d) for d in drop)}, tok)
    return m, cfg, tok, sd


@pytest.fixture(scope="module", params=["tiny", "small"])
def model(request):
    m, cfg, tok, sd = make_model(request.param)
    yield request.param, m, cfg, tok, sd
    m.engine.close()


def _wavs(n, T, g, zero_after=None):
    w = torch.randn(n, T, generator=g) * 0.05
    if zero_after is not None:
        w[-1, zero_after:] = 0
    return w


def _means(eng, wavs, workspace_bytes=None):
    n, T = wavs.shape
    mean = torch.full((n, eng.voice_frames(T), 64), float("nan"), device=eng.device)
    emb = eng.voice_encode(wavs, torch.zeros(n), None, mean_out=mean, workspace_bytes=workspace_bytes)
    torch.cuda.synchronize()
    return mean.cpu(), emb.cpu()


def test_encoder_mean_vs_oracle(model):
    """mean_out against `encoder_full` at every length class: one partial frame, just below / at a frame, several frames plus a tail,
    and a voice that is zero after 6407 samples inside a longer padded batch (encoded at the padded length, as the reference does)."""
    from oracle import vv_oracle as O
    preset, m, cfg, tok, sd = model
    tc = cfg.acoustic_tokenizer_config
    g = torch.Generator().manual_seed(5)
    worst = 0.0
    for n in (1, 2, 5):
        for T in (100, 3199, 3200, 3 * 3200 + 100, 5 * 3200 + 1):
            wavs = _wavs(n, T, g, zero_after=6407 if (n > 1 and T > 6407) else None)
            got, _ = _means(m.engine, wavs)
            want = O.encoder_full(sd, tc, wavs[:, None, :], ENC)
            assert got.shape == want.shape == (n, -(-T // 3200), 64)
            for v in range(n):
                e = rel_l2(got[v], want[v])
                worst = max(worst, e)
                assert e < 1e-4, (preset, n, T, v, e)
    report("voice_encoder_mean", preset=preset, max_rel_l2=worst)


@pytest.mark.parametrize("preset", ["1.5b-l2", "7b-l2"])
def test_full_width_encoder_and_connector(preset):
    """The shipped encoder widths (32 ... 2048 channels, depths 3-3-3-3-3-3-8) on 10 s voices, the second one ragged, at H = 1536 / 3584:
    the mean and the connected embeddings against the fp32 oracle run on the GPU with TF32 off."""
    from oracle import vv_oracle as O
    m, cfg, tok, sd = make_model(preset)
    try:
        g = torch.Generator().manual_seed(6)
        T = 240000
        wavs = _wavs(2, T, g, zero_after=171111)
        F = m.engine.voice_frames(T)
        masks = torch.ones(2, F, dtype=torch.bool)
        masks[1, -(F // 3):] = False
        noise = (torch.randn(2, generator=g), torch.randn(2, F, 64, generator=g))
        scale, bias = float(sd["model.speech_scaling_factor"]), float(sd["model.speech_bias_factor"])
        got_emb = m._voice(wavs, masks, scale, bias, noise=noise).cpu()
        got_mean, _ = _means(m.engine, wavs)
        keep = ("model.acoustic_", "model.speech_")
        w = {k: v.cuda() for k, v in sd.items() if k.startswith(keep)}
        tf32 = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            with torch.backends.cudnn.flags(enabled=True, allow_tf32=False), torch.no_grad():
                want_mean = O.encoder_full(w, cfg.acoustic_tokenizer_config, wavs.cuda()[:, None, :], ENC).cpu()
                want_emb = O.voice_prompt_embeds(w, cfg, wavs.cuda(), masks.cuda(), noise=(noise[0].cuda(), noise[1].cuda())).cpu()
        finally:
            torch.backends.cuda.matmul.allow_tf32 = tf32
        e_mean = [rel_l2(got_mean[v], want_mean[v]) for v in range(2)]
        e_emb = rel_l2(got_emb, want_emb)
        report("voice_full_width", preset=preset, mean_rel_l2=e_mean, embeds_rel_l2=e_emb)
        assert max(e_mean) < 1e-3 and e_emb < 1e-3, (e_mean, e_emb)
    finally:
        m.engine.close()


@pytest.mark.parametrize("mode", ["gaussian", "fix", "none"])
def test_sampling_modes_and_device_rng(model, mode):
    """All three std_dist_types with explicit noise, and the device-RNG draw order of `_voice(noise=None)`: std_n [n] then eps
    [n, F, vae_dim] (gaussian), eps only (fix), nothing (none)."""
    from oracle import vv_oracle as O
    preset, m, cfg, tok, sd = model
    tc = cfg.acoustic_tokenizer_config
    old = tc.std_dist_type
    tc.std_dist_type = mode
    try:
        g = torch.Generator().manual_seed(7)
        T = 2 * 3200 + 555
        wavs = _wavs(3, T, g)
        F = m.engine.voice_frames(T)
        masks = torch.rand(3, F, generator=g) < 0.7
        masks[:, 0] = True
        scale, bias = float(sd["model.speech_scaling_factor"]), float(sd["model.speech_bias_factor"])
        noise = (torch.randn(3, generator=g), torch.randn(3, F, 64, generator=g))
        got = m._voice(wavs, masks, scale, bias, noise=noise).cpu()
        want = O.voice_prompt_embeds(sd, cfg, wavs, masks, noise=noise)
        assert got.shape == want.shape == (int(masks.sum()), cfg.decoder_config.hidden_size)
        e = rel_l2(got, want)
        torch.manual_seed(99)
        got_rng = m._voice(wavs, masks, scale, bias).cpu()
        torch.manual_seed(99)
        std_n = torch.randn(3, device="cuda") if mode == "gaussian" else torch.zeros(3)
        eps = torch.randn(3, F, 64, device="cuda") if mode != "none" else torch.zeros(3, F, 64)
        want_rng = O.voice_prompt_embeds(sd, cfg, wavs, masks, noise=(std_n.cpu(), eps.cpu()))
        e_rng = rel_l2(got_rng, want_rng)
        report("voice_sampling", preset=preset, mode=mode, rel_l2=e, rng_rel_l2=e_rng)
        assert e < 1e-4 and e_rng < 1e-4, (e, e_rng)
        if mode != "none":
            assert rel_l2(got_rng, got) > 1e-3            # the noise really enters
    finally:
        tc.std_dist_type = old


def test_workspace_bounds(model):
    """The minimum workspace (one voice at a time, 64-row GEMM chunks) gives the result of a large one bit for bit (every row is computed
    by the same instructions whatever the grouping); one byte less is refused before anything is launched."""
    preset, m, cfg, tok, sd = model
    eng = m.engine
    g = torch.Generator().manual_seed(8)
    wavs = _wavs(3, 4 * 3200 + 17, g)
    need = eng.voice_workspace_bytes(3, wavs.shape[1])
    small_mean, small_emb = _means(eng, wavs, workspace_bytes=need)
    big_mean, big_emb = _means(eng, wavs, workspace_bytes=need * 8 + (64 << 20))
    assert torch.equal(small_mean, big_mean) and torch.equal(small_emb, big_emb)
    n, T = wavs.shape
    F = eng.voice_frames(T)
    wd, sig = wavs.cuda(), torch.zeros(n, device="cuda")
    out = torch.zeros(n, F, cfg.decoder_config.hidden_size, device="cuda")
    work = torch.empty(need, dtype=torch.uint8, device="cuda")
    P = lambda t: C.c_void_p(t.data_ptr())
    launches = eng.launch_count()
    rc = eng.lib.vv_voice_encode(eng.h, P(wd), n, T, P(sig), None, None, P(out), P(work), need - 1, eng.s)
    assert rc == -1 and "minimum" in eng.lib.vv_last_error().decode()
    assert eng.launch_count() == launches
    assert eng.lib.vv_voice_encode_workspace(eng.h, 0, T) == -1


def test_weight_presence():
    """No encoder tensors: the checkpoint still finalizes, `vv_voice_encode` returns VV_ERR_STATE and a voice-prompt generate() raises.
    Part of the encoder: vv_finalize_weights fails naming a missing tensor."""
    m, cfg, tok, sd = make_model("tiny", drop=(ENC + ".",))
    try:
        eng = m.engine
        assert m._voice is None
        work = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
        x = torch.zeros(1, 3200, device="cuda")
        out = torch.zeros(1, 1, cfg.decoder_config.hidden_size, device="cuda")
        P = lambda t: C.c_void_p(t.data_ptr())
        assert eng.lib.vv_voice_encode(eng.h, P(x), 1, 3200, P(x), None, None, P(out), P(work), 1 << 20, eng.s) == -3
        assert eng.lib.vv_voice_encode_workspace(eng.h, 1, 3200) == -3
        ids = torch.full((1, 6), tok.speech_diffusion_id)
        with pytest.raises(NV.VVError, match="encoder"):
            m.generate(input_ids=ids, tokenizer=tok, is_prefill=True, speech_tensors=torch.zeros(1, 3200),
                       speech_masks=torch.ones(1, 1, dtype=torch.bool), speech_input_mask=torch.ones(1, 6, dtype=torch.bool),
                       max_new_tokens=2, show_progress_bar=False)
    finally:
        m.engine.close()
    missing = ENC + ".stages.2.0.ffn.linear1.bias"
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    cfg = preset_config("tiny")
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, SEED, torch.bfloat16)
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=1)
    try:
        with pytest.raises(NV.VVError, match=missing.replace(".", r"\.")):
            m.load_state_dict({k: v for k, v in sd.items() if k != missing}, tok)
    finally:
        m.engine.close()


def _scripted(tok, plan):
    d = dict(d=tok.speech_diffusion_id, e=tok.speech_end_id, s=tok.speech_start_id, x=tok.eos_token_id)
    return [d[c] for c in plan]


@pytest.mark.parametrize("torch_prefill", [False, True])
def test_generate_voice_prompt_decode_prefill(torch_prefill):
    """Voice prompts through the token-by-token prefill (`torch_prefill=False`, and `prefill_impl="decode"` on a model that keeps the
    PyTorch prefill): B = 1, and B = 2 ragged left-padded prompts with one and two voices.  Tokens exact, audio within 1e-2 of the
    oracle fed the oracle's own voice embeddings."""
    from oracle import vv_oracle as O
    from vibevoice_b200.modeling import ForcedTokenScript
    m, cfg, tok, sd = make_model("tiny", max_batch=2, torch_prefill=torch_prefill)
    try:
        dc = cfg.decoder_config
        g = torch.Generator().manual_seed(9)
        scale, bias = float(sd["model.speech_scaling_factor"]), float(sd["model.speech_bias_factor"])
        T = 3 * 3200 + 100
        F = 4
        wavs = _wavs(3, T, g)
        wavs[1, 2 * 3200 + 7:] = 0
        vmask = torch.zeros(3, F, dtype=torch.bool)
        vmask[0, :4] = True
        vmask[1, :3] = True
        vmask[2, :2] = True
        noise = (torch.randn(3, generator=g), torch.randn(3, F, 64, generator=g))
        want_emb = O.voice_prompt_embeds(sd, cfg, wavs, vmask, noise=noise)
        L0 = 24
        for B in (1, 2):
            nv = 1 if B == 1 else 3
            ids = torch.randint(0, dc.vocab_size - 20, (B, L0), generator=g)
            ids[:, -1] = tok.speech_start_id
            mask = torch.ones(B, L0, dtype=torch.long)
            sim = torch.zeros(B, L0, dtype=torch.bool)
            sim[0, 3:7] = True                                    # voice 0: 4 frames
            if B == 2:
                mask[1, :5] = 0
                ids[1, :5] = tok.pad_token_id
                sim[1, 7:10] = True                               # voice 1: 3 frames
                sim[1, 13:15] = True                              # voice 2: 2 frames
            ids[sim] = tok.speech_diffusion_id
            counts = sim.sum(-1).tolist()
            offs = [0, counts[0], counts[0] + (counts[1] if B == 2 else 0)]
            emb = want_emb[: offs[B]]
            scripts = [_scripted(tok, "dddx"), _scripted(tok, "ddesdx")][:B]
            m.set_ddpm_inference_steps(5)
            torch.manual_seed(0)
            out = m.generate(input_ids=ids, attention_mask=mask, tokenizer=tok, cfg_scale=1.3, is_prefill=True, speech_tensors=wavs[:nv],
                             speech_masks=vmask[:nv], speech_input_mask=sim, _voice_noise=(noise[0][:nv], noise[1][:nv]),
                             logits_processor=[ForcedTokenScript(scripts)], max_new_tokens=12, show_progress_bar=False,
                             prefill_impl="decode")
            torch.manual_seed(0)
            ref = O.generate(sd, cfg, ids, mask, tok, cfg_scale=1.3, num_steps=5, max_new_tokens=12, forced_tokens=scripts, kv_bf16=True,
                             speech_embeds=[(sim[r][mask[r].bool()], emb[offs[r]:offs[r + 1]]) for r in range(B)])
            assert torch.equal(out.sequences, ref.sequences)
            assert torch.equal(out.reach_max_step_sample, ref.reach_max_step_sample)
            for r in range(B):
                a, b = out.speech_outputs[r].cpu(), ref.speech_outputs[r]
                assert a.shape == b.shape
                e = rel_l2(a, b)
                report("generate_voice_decode_prefill", torch_prefill=torch_prefill, B=B, row=r, audio_rel_l2=e)
                assert e < 1e-2, (B, r, e)
    finally:
        m.engine.close()
