"""`-m gpu`: 9..16 prompts per GPU (max_batch 9..16, 2B = 18..32 sequences) at every preset width.

At B >= 9 the LM and sampler programs hold 18..32 rows (MMA height 64, operand rows [0, 32) hi and [32, 64) lo), the codec stages with
T > 2 frames leave the stream program for the kernel-per-stage path, and the connectors run in two row groups of at most 8.  Stages whose
activation operand needs more shared memory than the weight ring leaves run as K slices: at 1.5B the LM gate/up projection (two slices);
at 7B the sampler's gate/up (three) and down (two) linears, the LM's gate/up and down projections (three each) and the o-projection with
its attention merge (two slices at B <= 11, three at 12..14, four at 15..16: the per-(row, head) merge table holds 128 entries, so at
32 rows one slice takes at most four heads).
Tolerances as in test_gpu_presets.py (2e-4 sampler latents, 2e-3 codec frames and LM hidden states) and test_gpu_queue.py (audio)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from test_gpu_parity import rel_l2, report
from test_gpu_presets import _codec_checks, _lm_checks, _model, _sampler_checks, _state
from test_gpu_queue import check, make_model, requests, serve

PRESETS = ["tiny", "tiny64", "1.5b-l2", "7b-l2", "streaming-0.5b-l4"]
ODE, SDE = "dpmsolver++", "sde-dpmsolver++"


# ---- every preset at every batch size 9..16 --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", list(range(9, 17)))
@pytest.mark.parametrize("preset", PRESETS)
def test_every_preset_runs_at_b9_to_16(preset, B):
    """One LM decode, one sampler call, one codec decode, one semantic encode and one connector pass succeed and stay finite."""
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
        eng.connect()
        eng.sync()
        for name in ("hidden", "logits", "latent", "audio", "feat", "embeds"):
            t = getattr(eng, name)
            assert torch.isfinite(t).all(), (preset, B, name)
        assert eng.latent.abs().sum() > 0 and eng.audio.abs().sum() > 0
    finally:
        model.engine.close()


@pytest.mark.parametrize("preset", PRESETS)
def test_max_batch_17_is_refused(preset):
    from vibevoice_b200 import _native as N
    with pytest.raises(N.VVError, match=r"max_batch 17 outside \[1,16\]"):
        _model(preset, 17, oracle=False)


# ---- stream programs against the oracle ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("preset,B", [("1.5b-l2", 9), ("1.5b-l2", 12), ("1.5b-l2", 16), ("7b-l2", 9), ("7b-l2", 16)])
def test_sampler_vs_oracle_b16(preset, B):
    """The 10- and 30-step sampler programs, a ragged active set, and at B = 9 the SDE solver with injected step noise."""
    model, cfg, tok, sdf = _model(preset, B)
    try:
        _sampler_checks(model, cfg, sdf, B, preset, sde=(B == 9))
    finally:
        model.engine.close()


@pytest.mark.parametrize("preset", ["1.5b-l2", "7b-l2"])
def test_per_row_solver_b16(preset):
    """16 rows of the per-row sampler with 5 / 10 / 20 steps, ODE and SDE mixed: each row against the same row sampled alone with
    `set_diffusion_steps` and against the oracle."""
    from oracle import vv_oracle as O
    from vibevoice_b200.schedule import DPMSolverMultistepScheduler
    B = 16
    model, cfg, tok, sdf = _model(preset, B)
    try:
        eng = model.engine
        H = cfg.decoder_config.hidden_size
        g = torch.Generator().manual_seed(1600 + H)
        cond = torch.randn(2 * B, H, generator=g)
        noise = torch.randn(B, 64, generator=g)
        step_noise = [torch.randn(20, 64, generator=g) for _ in range(B)]
        settings = [([5, 10, 20][r % 3], [1.3, 1.0, 2.5, 1.5][r % 4], [ODE, SDE][(r // 2) % 2]) for r in range(B)]
        sched = lambda solver: DPMSolverMultistepScheduler.from_config(eng.scheduler.config, algorithm_type=solver)
        solo = []
        for r, (steps, cs, solver) in enumerate(settings):
            eng.sampler_per_row(0)
            eng.set_scheduler(sched(solver))
            eng.set_diffusion_steps(steps)
            with torch.cuda.stream(eng.stream):
                eng.hidden.copy_(cond.cuda())
            eng.upload_frame_inputs(noise[r:r + 1], [r])
            if solver == SDE:
                eng.upload_step_noise(lambda i: step_noise[r][i:i + 1], [r])
            eng.diffusion_sample(cs)
            eng.sync()
            solo.append(eng.latent[r].cpu().clone())
        eng.sampler_per_row(20)
        for r, (steps, cs, solver) in enumerate(settings):
            eng.set_row_sampler(r, steps, solver, cs)
            if solver == SDE:
                eng.upload_row_step_noise(r, step_noise[r][:steps])
        with torch.cuda.stream(eng.stream):
            eng.hidden.copy_(cond.cuda())
        eng.upload_frame_inputs(noise, list(range(B)))
        eng.diffusion_sample(1.0)
        eng.sync()
        got = eng.latent.cpu().clone()
        eng.sampler_per_row(0)
        for r, (steps, cs, solver) in enumerate(settings):
            kw = dict(algorithm_type=solver, step_noise=[step_noise[r][i:i + 1] for i in range(steps)]) if solver == SDE else {}
            want = O.sample_speech_tokens(sdf, cond[r:r + 1], cond[B + r:B + r + 1], cs, steps,
                                          torch.cat([noise[r:r + 1], torch.zeros(1, 64)]), **kw)[0]
            es, eo = rel_l2(got[r], solo[r]), rel_l2(got[r], want)
            report("sampler_rows_b16", preset=preset, row=r, settings=settings[r], vs_solo=es, vs_oracle=eo)
            assert es < 2e-4 and eo < 2e-4, (r, settings[r], es, eo)
    finally:
        model.engine.close()


@pytest.mark.parametrize("B", [9, 16])
def test_streaming_codec_vs_oracle_b16(B):
    """Decoder + semantic encoder over 12 frames with ragged active sets and a state zeroing of rows 0 and B - 1 (>= 8) in the middle."""
    model, cfg, tok, sdf = _model("1.5b-l2", B)
    try:
        _codec_checks(model, cfg, sdf, B, "1.5b-l2")
    finally:
        model.engine.close()


def _lm_lens(B, seed):
    g = torch.Generator().manual_seed(seed)
    pos = [16500] + [int(x) for x in torch.randint(60, 2200, (B - 1,), generator=g)]
    neg = [int(x) for x in torch.randint(0, 140, (B,), generator=g)]
    neg[1] = 64                                              # page edges
    neg[2] = 63
    return pos, neg


@pytest.mark.parametrize("preset,B", [("1.5b-l2", 9), ("1.5b-l2", 16), ("7b-l2", 16)])
def test_lm_decode_vs_oracle_b16(preset, B):
    """Ragged positive and negative contexts (one positive row at 16 500 tokens, negative rows on both sides of a page edge), 4 decode
    steps with the negative rows advancing every other step."""
    model, cfg, tok, sdf = _model(preset, B)
    try:
        pos, neg = _lm_lens(B, B)
        _lm_checks(model, cfg, sdf, B, preset, pos, neg)
    finally:
        model.engine.close()


# ---- sequences 16..31 ------------------------------------------------------------------------------------------------------------------
def test_sequences_16_to_31():
    """kv_set_len, kv_commit, kv_delete and set_row_mode on the negative sequences of rows 8..15 (sequences 24..31), then decode only those
    against the oracle.  The other sequences keep their lengths and cache entries, and NaN / +-1e4 inputs in their rows do not leak."""
    from oracle import vv_oracle as O
    from test_gpu_scale import _structured_kv
    B = 16
    model, cfg, tok, sdf = _model("1.5b-l2", B)
    try:
        eng = model.engine
        dc = cfg.decoder_config
        nl, nkv, hd, H = dc.num_hidden_layers, dc.num_key_value_heads, dc.head_dim, dc.hidden_size
        eng.kv_init(8192)
        g = torch.Generator().manual_seed(31)
        lens = [40 + 7 * s for s in range(2 * B)]
        caches = [O.KVCache(nl, kv_bf16=True) for _ in range(2 * B)]
        for seq, L in enumerate(lens):
            eng.kv_set_len(seq, 0)
            for layer in range(nl):
                k, v = _structured_kv(nkv, L, hd, g)
                caches[seq].preload(layer, k.float(), v.float())
                with torch.cuda.stream(eng.stream):
                    eng.kv_write(seq, layer, 0, k.transpose(0, 1).contiguous().cuda(), v.transpose(0, 1).contiguous().cuda())
                eng.sync()
            eng.kv_set_len(seq, L)
        live = list(range(24, 32))
        # kv_set_len: shrink 24 and 25; kv_delete: forget position 5 of 26 (its last entry moves there)
        for s, n in ((24, lens[24] - 9), (25, 64)):
            eng.kv_set_len(s, n)
            caches[s].truncate(n)
            lens[s] = n
        eng.kv_delete(26, 5)
        for layer in range(nl):
            c = caches[26]
            c.k[layer][:, 5] = c.k[layer][:, lens[26] - 1]
            c.v[layer][:, 5] = c.v[layer][:, lens[26] - 1]
        caches[26].truncate(lens[26] - 1)
        lens[26] -= 1
        before = {s: eng.kv_read(s, 0, 0, lens[s]) for s in (0, 15, 16, 23)}
        eng.set_row_mode([1 if s in live else 0 for s in range(2 * B)])
        try:
            for step in range(3):
                x = torch.randn(2 * B, H, generator=g) * 0.05
                for s in range(2 * B):
                    if s not in live:
                        x[s] = [float("nan"), 1e4, -1e4][s % 3]
                with torch.cuda.stream(eng.stream):
                    eng.embeds.copy_(x.cuda())
                eng.lm_decode()
                eng.read_tokens()
                adv = [1 if (s in live and (step == 0 or s % 2 == 0)) else 0 for s in range(2 * B)]
                got = eng.hidden.cpu()
                for s in live:
                    n0 = len(caches[s])
                    want = O.qwen2_forward(sdf, dc, x[s][None], caches[s], n0)[0]
                    if not adv[s]:
                        caches[s].truncate(n0)
                    e = rel_l2(got[s], want)
                    report("seq16_31", step=step, seq=s, rel_l2=e)
                    assert torch.isfinite(got[s]).all() and e < 2e-3, (step, s, e)
                eng.kv_commit(adv)
                for s in live:
                    lens[s] += adv[s]
                    assert eng.kv_len(s) == lens[s], s
        finally:
            eng.set_row_mode([1] * (2 * B))
        for s in range(2 * B):
            assert eng.kv_len(s) == lens[s], s
        for s, (k0, v0) in before.items():
            k1, v1 = eng.kv_read(s, 0, 0, lens[s])
            assert torch.equal(k0, k1) and torch.equal(v0, v1), s
    finally:
        model.engine.close()


# ---- connectors ------------------------------------------------------------------------------------------------------------------------
def _connector64(sd, p, x):
    f = lambda n: sd[n].double()
    y = x.double() @ f(p + ".fc1.weight").T + f(p + ".fc1.bias")
    y = y * torch.rsqrt(y.pow(2).mean(-1, keepdim=True) + 1e-6) * f(p + ".norm.weight")
    return y @ f(p + ".fc2.weight").T + f(p + ".fc2.bias")


@pytest.mark.parametrize("B", [9, 16])
def test_connectors_vs_float64_b16(B):
    """Both connectors over B rows in groups of at most 8 against a float64 reference; select_embeds copies the active rows into both
    streams and leaves inactive rows as they were."""
    model, cfg, tok, _ = _model("1.5b-l2", B, oracle=False)
    try:
        sd = _state("1.5b-l2")["sd"]
        eng = model.engine
        H, S = cfg.decoder_config.hidden_size, cfg.semantic_vae_dim
        g = torch.Generator().manual_seed(B)
        lat, sem = torch.randn(B, 64, generator=g), torch.randn(B, S, generator=g)
        active = [r for r in range(B) if r % 4 != 2]
        with torch.cuda.stream(eng.stream):
            eng.latent.copy_(lat.cuda()); eng.feat.copy_(sem.cuda()); eng.embeds.fill_(7.0)
        eng.upload_frame_inputs(torch.zeros(len(active), 64), active)
        eng.connect()
        eng.sync()
        want = _connector64(sd, "model.acoustic_connector", lat) + _connector64(sd, "model.semantic_connector", sem)
        emb = eng.embeds.cpu()
        for r in range(B):
            if r in active:
                e = max(rel_l2(emb[r], want[r]), rel_l2(emb[B + r], want[r]))
                report("connectors_b16", B=B, row=r, rel_l2=e)
                assert e < 1e-4, (r, e)
            else:
                assert torch.all(emb[r] == 7.0) and torch.all(emb[B + r] == 7.0), r
    finally:
        model.engine.close()


# ---- closed loop -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("preset,steps", [("tiny", 5), ("1.5b-l2", 5)])
def test_generate_16_ragged_prompts_vs_oracle(preset, steps):
    """generate() with 16 ragged left-padded prompts, scripted speaker turns and per-row EOS, against the oracle: sequences, finished
    rows and reach_max_step_sample exact, audio within the closed-loop tolerance."""
    from oracle import vv_oracle as O
    from vibevoice_b200.modeling import ForcedTokenScript
    B = 16
    model, cfg, tok, sdf = _model(preset, B)
    try:
        dc = cfg.decoder_config
        g = torch.Generator().manual_seed(16)
        L0 = 14
        ids = torch.randint(0, dc.vocab_size - 20, (B, L0), generator=g)
        ids[:, -1] = tok.speech_start_id
        mask = torch.ones(B, L0, dtype=torch.long)
        for r in range(B):
            pad = r % 6
            mask[r, :pad] = 0
            ids[r, :pad] = tok.pad_token_id
        m = dict(d=tok.speech_diffusion_id, e=tok.speech_end_id, s=tok.speech_start_id, x=tok.eos_token_id)
        plans = ["ddx", "desddx", "dddx", "ddesdx", "dx", "dddesdx"]
        scripts = [[m[c] for c in plans[r % len(plans)]] for r in range(B)]
        model.set_ddpm_inference_steps(steps)
        torch.manual_seed(0)
        out = model.generate(input_ids=ids, attention_mask=mask, tokenizer=tok, cfg_scale=1.3, is_prefill=False,
                             logits_processor=[ForcedTokenScript(scripts)], max_new_tokens=10, show_progress_bar=False)
        torch.manual_seed(0)
        ref = O.generate(sdf, cfg, ids, mask, tok, cfg_scale=1.3, num_steps=steps, max_new_tokens=10, forced_tokens=scripts, kv_bf16=True)
        assert torch.equal(out.sequences, ref.sequences)
        assert torch.equal(out.reach_max_step_sample, ref.reach_max_step_sample)
        for r in range(B):
            a, b = out.speech_outputs[r].cpu(), ref.speech_outputs[r]
            assert a.shape == b.shape == (1, 3200 * scripts[r].count(tok.speech_diffusion_id)), r
            e = rel_l2(a, b)
            report("generate_b16", preset=preset, row=r, audio_rel_l2=e)
            assert e < 1e-2, (r, e)
    finally:
        model.engine.close()


# ---- request queue ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("preset,n", [("tiny", 32), ("1.5b-l2", 24)])
def test_queue_at_max_batch_16(preset, n):
    """n requests of mixed lengths, steps, CFG scales and solvers (every third with a voice prompt) over 16 rows: every request equals
    torch.manual_seed(seed) + its solo generate()."""
    m, cfg, tok = make_model(preset, 16, prefill_impl="native")
    try:
        reqs = requests(cfg, tok, n, 16, seed=16, voices=preset == "tiny")
        got, rows = serve(m, reqs)
        assert [p[2] for p in rows] == [r["inputs"]["input_ids"].shape[1] for r in reqs]
        assert [p[0] for p in rows[:16]] == list(range(16))
        check(m, tok, reqs, got)
    finally:
        m.engine.close()
