"""`-m gpu` parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.

Tolerances (stated here, north_star: "within a stated fp tolerance; bit-exact for token/index bookkeeping"):
  * weights are bf16 on both sides (the oracle up-casts the same bf16 values), activations fp32, accumulation
    fp32 -> the only differences are summation order and fast-math exp: stage outputs must agree to
    rel-L2 <= 2e-4 (single stage) / 2e-3 (28-layer LM with a bf16 KV cache, audio after 26 codec blocks);
  * token ids / sequence bookkeeping / finished flags: exact.
"""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from vibevoice_b200 import _native as NV
from vibevoice_b200.configuration import preset_config
from vibevoice_b200.synth import SynthTokenizer, synth_state_dict

SEED = 1234
# per-test error figures, appended as JSON lines (VV_REPORT_DIR, default reports/ in the repository)
OUT = os.environ.get("VV_REPORT_DIR") or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "reports")


def rel_l2(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def report(name, **kv):
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "parity_report.jsonl"), "a") as f:
        f.write(json.dumps(dict(test=name, **kv)) + "\n")


def make_model(preset, max_batch):
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    cfg = preset_config(preset)
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, SEED, torch.bfloat16)
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=max_batch)
    m.load_state_dict(sd, tok)
    return m, cfg, tok, sd


@pytest.fixture(scope="module")
def tiny2():
    m, cfg, tok, sd = make_model("tiny", 2)
    yield m, cfg, tok, sd
    m.engine.close()


@pytest.fixture(scope="module")
def small1():
    m, cfg, tok, sd = make_model("small", 1)
    yield m, cfg, tok, sd
    m.engine.close()


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K", [(1, 64, 256), (2, 1536, 1536), (2, 2048, 1536), (2, 4608, 1536), (2, 1536, 8960),
                                   (4, 320, 448), (8, 1024, 2048), (3, 100, 264), (16, 512, 1024), (2, 64, 18944),
                                   (40, 2048, 512), (200, 1024, 256), (70, 96, 40)])
def test_gemv_matches_torch(tiny2, M, N, K):
    """The weight-streaming GEMV / tiled GEMM against a plain PyTorch fp32 reference of the same op."""
    import ctypes as C
    eng = tiny2[0].engine
    g = torch.Generator().manual_seed(M * 1000003 + N * 101 + K)
    W = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    x = torch.randn(M, K, generator=g)
    bias = torch.randn(N, generator=g) * 0.1
    nw = torch.rand(K, generator=g) + 0.5
    Wd, xd, bd, nwd = W.cuda(), x.cuda(), bias.cuda(), nw.cuda()
    P = lambda t: C.c_void_p(t.data_ptr())
    cases = [(NV.PRO_NONE, NV.EPI_NONE), (NV.PRO_NONE, NV.EPI_GELU), (NV.PRO_NONE, NV.EPI_SILU), (NV.PRO_RMSNORM, NV.EPI_GELU),
             (NV.PRO_SILU, NV.EPI_NONE), (NV.PRO_RMSNORM, NV.EPI_SWIGLU), (NV.PRO_NONE, NV.EPI_RESID)]
    for pro, epi in cases:
        if epi == NV.EPI_SWIGLU and N % 2:
            continue
        y = torch.full((M, N // 2 if epi == NV.EPI_SWIGLU else N), 0.25, device="cuda")
        y0 = y.clone()
        with torch.cuda.stream(eng.stream):
            NV.check(eng.lib.vv_debug_gemv(eng.h, P(Wd), P(bd), P(xd), P(y), M, N, K, pro, P(nwd), 1e-5, epi, eng.s))
        eng.sync()
        xt = x.clone()
        if pro == NV.PRO_RMSNORM:
            xt = xt * torch.rsqrt(xt.pow(2).mean(-1, keepdim=True) + 1e-5) * nw
        elif pro == NV.PRO_SILU:
            xt = torch.nn.functional.silu(xt)
        ref = xt @ W.float().T + bias
        if epi == NV.EPI_GELU:
            ref = torch.nn.functional.gelu(ref)
        elif epi == NV.EPI_SILU:
            ref = torch.nn.functional.silu(ref)
        elif epi == NV.EPI_SWIGLU:
            ref = torch.nn.functional.silu(ref[:, 0::2]) * ref[:, 1::2]
        elif epi == NV.EPI_RESID:
            ref = ref + y0.cpu()
        e = rel_l2(y, ref)
        report("gemv", M=M, N=N, K=K, pro=pro, epi=epi, rel_l2=e)
        assert e < 2e-5, (M, N, K, pro, epi, e)


def _run_sampler(model, cfg, sd, pos, neg, noise_rows, active_rows, cfg_scale, steps):
    eng = model.engine
    B = eng.B
    eng.set_diffusion_steps(steps)
    hid = torch.zeros(2 * B, cfg.decoder_config.hidden_size)
    for i, r in enumerate(active_rows):
        hid[r], hid[B + r] = pos[i], neg[i]
    with torch.cuda.stream(eng.stream):
        eng.hidden.copy_(hid.cuda())
    eng.upload_frame_inputs(noise_rows, active_rows)
    eng.diffusion_sample(cfg_scale)
    eng.sync()
    return eng.latent.cpu()[active_rows]


@pytest.mark.parametrize("steps,cfg_scale", [(5, 1.5), (10, 1.3), (30, 1.3)])
def test_diffusion_sampler_vs_oracle(tiny2, steps, cfg_scale):
    from oracle import vv_oracle as O
    model, cfg, tok, sd = tiny2
    H = cfg.decoder_config.hidden_size
    g = torch.Generator().manual_seed(steps)
    pos, neg = torch.randn(2, H, generator=g), torch.randn(2, H, generator=g)
    noise = torch.randn(4, 64, generator=g)
    got = _run_sampler(model, cfg, sd, pos, neg, noise[:2], [0, 1], cfg_scale, steps)
    want = O.sample_speech_tokens(sd, pos, neg, cfg_scale, steps, noise)
    e = rel_l2(got, want)
    report("sampler", steps=steps, rel_l2=e)
    assert e < 2e-4, e
    # ragged: only row 1 active; row 0 must not influence it
    got1 = _run_sampler(model, cfg, sd, pos[1:], neg[1:], noise[1:2], [1], cfg_scale, steps)
    want1 = O.sample_speech_tokens(sd, pos[1:], neg[1:], cfg_scale, steps, noise[1:2].repeat(2, 1))
    assert rel_l2(got1, want1) < 2e-4


def test_golden_sampler_fixture(golden, tiny2):
    """Committed golden vectors produced by the reference's own `sample_speech_tokens` (tests/golden/head.pt)."""
    model, cfg, tok, sd_bf16 = tiny2
    g = golden("head")
    # the fixture was produced with fp32 weights; the engine holds their bf16 rounding -> compare through the oracle
    from oracle import vv_oracle as O
    for n_steps, s in g["samples"].items():
        got = _run_sampler(model, cfg, sd_bf16, s["pos"], s["neg"], s["noise"][:2], [0, 1], s["cfg_scale"], n_steps)
        want_bf16w = O.sample_speech_tokens(sd_bf16, s["pos"], s["neg"], s["cfg_scale"], n_steps, s["noise"])
        assert rel_l2(got, want_bf16w) < 2e-4
        # and the bf16-weight result stays close to the reference's fp32-weight golden latent
        e = rel_l2(got, s["latent"])
        report("sampler_golden", steps=n_steps, rel_l2_vs_fp32_reference=e)
        assert e < 5e-2


def test_streaming_codec_vs_oracle(tiny2):
    """Decoder + semantic encoder over several frames with ragged active rows and a <speech_end> state zeroing."""
    from oracle import vv_oracle as O
    model, cfg, tok, sd = tiny2
    eng = model.engine
    eng.codec_state_reset()
    a, s = O.StreamState(2), O.StreamState(2)
    g = torch.Generator().manual_seed(5)
    script = [[0, 1], [0], [0, 1], [1], [0, 1], [0, 1]]
    zero_before = {4: [0]}
    scale, bias = float(sd["model.speech_scaling_factor"]), float(sd["model.speech_bias_factor"])
    worst_a = worst_s = 0.0
    for f, rows in enumerate(script):
        if f in zero_before:
            eng.codec_state_zero(zero_before[f]); a.set_to_zero(zero_before[f]); s.set_to_zero(zero_before[f])
        lat = torch.randn(len(rows), 64, generator=g)
        full = torch.zeros(2, 64)
        full[rows] = lat
        with torch.cuda.stream(eng.stream):
            eng.latent.copy_(full.cuda())
        eng.upload_frame_inputs(torch.zeros(len(rows), 64), rows)
        eng.codec_decode()
        eng.semantic_encode()
        eng.sync()
        audio = O.decoder_frame(sd, cfg.acoustic_tokenizer_config, (lat / scale - bias)[:, None, :], a, rows)
        sem = O.encoder_frame(sd, cfg.semantic_tokenizer_config, audio, s, rows)
        ea = rel_l2(eng.audio.cpu()[rows], audio[:, 0])
        es = rel_l2(eng.feat.cpu()[rows], sem[:, 0])
        worst_a, worst_s = max(worst_a, ea), max(worst_s, es)
        report("codec", frame=f, rows=rows, audio_rel_l2=ea, sem_rel_l2=es)
    assert worst_a < 2e-3 and worst_s < 2e-3, (worst_a, worst_s)


def test_connectors_vs_oracle(tiny2):
    from oracle import vv_oracle as O
    model, cfg, tok, sd = tiny2
    eng = model.engine
    g = torch.Generator().manual_seed(9)
    lat, sem = torch.randn(2, 64, generator=g), torch.randn(2, 128, generator=g)
    with torch.cuda.stream(eng.stream):
        eng.latent.copy_(lat.cuda()); eng.feat.copy_(sem.cuda()); eng.embeds.fill_(7.0)
    eng.upload_frame_inputs(torch.zeros(1, 64), [1])
    eng.connect()
    eng.sync()
    want = O.connector(sd, "model.acoustic_connector", lat) + O.connector(sd, "model.semantic_connector", sem)
    emb = eng.embeds.cpu()
    assert rel_l2(emb[1], want[1]) < 2e-4 and rel_l2(emb[3], want[1]) < 2e-4     # row 1 active -> rows 1 and B+1
    assert torch.all(emb[0] == 7.0) and torch.all(emb[2] == 7.0)                  # inactive row keeps its token embedding


def _lm_roundtrip(model, cfg, tok, sd, n_prompt, n_steps):
    from oracle import vv_oracle as O
    eng = model.engine
    dc = cfg.decoder_config
    B = eng.B
    if eng.kv_pages == 0:
        eng.kv_init(4096)
    for s_ in range(2 * B):
        eng.kv_set_len(s_, 0)
    g = torch.Generator().manual_seed(77)
    ids = torch.randint(0, dc.vocab_size - 20, (B, n_prompt), generator=g)
    embw = sd["model.language_model.embed_tokens.weight"]
    caches = [O.KVCache(dc.num_hidden_layers, kv_bf16=True) for _ in range(2 * B)]
    errs = []
    for t in range(n_prompt + n_steps):
        if t < n_prompt:
            toks = ids[:, t].tolist()
            eng.embed_tokens(toks + toks, eng.embeds)
            x = torch.cat([embw[ids[:, t]].float(), embw[ids[:, t]].float()])
        else:
            x = torch.randn(2 * B, dc.hidden_size, generator=g) * 0.05
            with torch.cuda.stream(eng.stream):
                eng.embeds.copy_(x.cuda())
        eng.lm_decode()
        toks_dev, logits_dev = eng.read_tokens()
        adv = [1] * B + [1 if t % 2 == 0 else 0] * B          # negative rows advance every other step
        want = []
        for r in range(2 * B):
            n0 = len(caches[r])
            h = O.qwen2_forward(sd, dc, x[r][None], caches[r], n0)
            if not adv[r]:
                caches[r].truncate(n0)
            want.append(h[0])
        want = torch.stack(want)
        eng.kv_commit(adv)
        errs.append(rel_l2(eng.hidden.cpu(), want))
        valid = sorted({tok.speech_start_id, tok.speech_end_id, tok.speech_diffusion_id, tok.eos_token_id})
        lw = want[:B] @ O.lm_head_weight(sd, dc)[valid].float().T
        assert rel_l2(torch.from_numpy(logits_dev.copy()), lw) < 5e-3
        margin = lw.sort(dim=-1).values
        for r in range(B):
            if float(margin[r, -1] - margin[r, -2]) > 1e-3 * float(lw[r].abs().max()):
                assert int(toks_dev[r]) == valid[int(lw[r].argmax())]
    return errs


def test_lm_decode_vs_oracle(tiny2):
    model, cfg, tok, sd = tiny2
    errs = _lm_roundtrip(model, cfg, tok, sd, n_prompt=70, n_steps=6)     # crosses a 64-token page and a 32-token tile
    report("lm_decode_tiny", max_rel_l2=max(errs))
    assert max(errs) < 2e-3, errs


def test_lm_decode_small_vs_oracle(small1):
    model, cfg, tok, sd = small1
    errs = _lm_roundtrip(model, cfg, tok, sd, n_prompt=40, n_steps=4)
    report("lm_decode_small", max_rel_l2=max(errs))
    assert max(errs) < 2e-3, errs


def _scripted(tok, plan):
    m = dict(d=tok.speech_diffusion_id, e=tok.speech_end_id, s=tok.speech_start_id, x=tok.eos_token_id)
    return [m[c] for c in plan]


def test_generate_loop_vs_oracle_forced_script(tiny2):
    """Closed loop, B=2, ragged left-padded prompts, a scripted token sequence with a speaker turn (<end>,<start>):
    exercises negative-stream restart, codec-state zeroing, per-row finishing.  Bookkeeping exact, audio close."""
    from oracle import vv_oracle as O
    from vibevoice_b200.modeling import ForcedTokenScript
    model, cfg, tok, sd = tiny2
    dc = cfg.decoder_config
    g = torch.Generator().manual_seed(3)
    L0 = 12
    ids = torch.randint(0, dc.vocab_size - 20, (2, L0), generator=g)
    ids[:, -1] = tok.speech_start_id
    mask = torch.ones(2, L0, dtype=torch.long)
    mask[1, :4] = 0
    ids[1, :4] = tok.pad_token_id
    scripts = [_scripted(tok, "dddesddx"), _scripted(tok, "ddddddddx")]
    model.set_ddpm_inference_steps(5)
    torch.manual_seed(0)
    out = model.generate(input_ids=ids, attention_mask=mask, tokenizer=tok, cfg_scale=1.3, is_prefill=False,
                         logits_processor=[ForcedTokenScript(scripts)], max_new_tokens=40, show_progress_bar=False)
    torch.manual_seed(0)
    ref = O.generate(sd, cfg, ids, mask, tok, cfg_scale=1.3, num_steps=5, max_new_tokens=40, forced_tokens=scripts, kv_bf16=True)
    assert torch.equal(out.sequences, ref.sequences)                                   # bit-exact token bookkeeping
    assert torch.equal(out.reach_max_step_sample, ref.reach_max_step_sample)
    for r in range(2):
        a, b = out.speech_outputs[r].cpu(), ref.speech_outputs[r]
        assert a.shape == b.shape == (1, 3200 * scripts[r].count(tok.speech_diffusion_id))
        e = rel_l2(a, b)
        report("generate_forced", row=r, audio_rel_l2=e)
        assert e < 1e-2, (r, e)


def test_generate_free_running_tokens(tiny2):
    """No forced tokens: the constrained argmax itself drives the state machine; the token sequence must match the oracle
    wherever the oracle's decision margin is not a numerical tie."""
    from oracle import vv_oracle as O
    model, cfg, tok, sd = tiny2
    dc = cfg.decoder_config
    g = torch.Generator().manual_seed(11)
    ids = torch.randint(0, dc.vocab_size - 20, (1, 9), generator=g)
    ids[:, -1] = tok.speech_start_id
    model.set_ddpm_inference_steps(5)
    torch.manual_seed(1)
    out = model.generate(input_ids=ids, tokenizer=tok, cfg_scale=1.3, is_prefill=False, max_new_tokens=10, show_progress_bar=False)
    torch.manual_seed(1)
    ref = O.generate(sd, cfg, ids, None, tok, cfg_scale=1.3, num_steps=5, max_new_tokens=10, kv_bf16=True, trace=True)
    margins = [float(l.sort(dim=-1).values[0, -1] - l.sort(dim=-1).values[0, -2]) for l in ref.trace["logits"]]
    report("generate_free", margins=margins, got=out.sequences.tolist(), want=ref.sequences.tolist())
    n = min(out.sequences.shape[1], ref.sequences.shape[1])
    first_tie = next((i for i, m in enumerate(margins) if m < 1e-3), len(margins))
    upto = min(n, ids.shape[1] + first_tie)
    assert torch.equal(out.sequences[:, :upto], ref.sequences[:, :upto])


def test_generate_do_sample_vs_oracle(tiny2):
    """`do_sample=True` (reference :493-496): multinomial over the constrained distribution.  Same generator seed on both sides;
    the probabilities differ by ~1e-4, so the draws must agree unless a uniform lands within that distance of a bin edge."""
    from oracle import vv_oracle as O
    model, cfg, tok, sd = tiny2
    dc = cfg.decoder_config
    g = torch.Generator().manual_seed(12)
    ids = torch.randint(0, dc.vocab_size - 20, (2, 7), generator=g)
    ids[:, -1] = tok.speech_start_id
    model.set_ddpm_inference_steps(4)
    agree = 0
    for seed in range(4):
        torch.manual_seed(3)
        out = model.generate(input_ids=ids, tokenizer=tok, cfg_scale=1.3, is_prefill=False, max_new_tokens=8, show_progress_bar=False,
                             generation_config={"do_sample": True, "top_k": 0}, sample_generator=torch.Generator().manual_seed(100 + seed))
        torch.manual_seed(3)
        ref = O.generate(sd, cfg, ids, None, tok, cfg_scale=1.3, num_steps=4, max_new_tokens=8, kv_bf16=True, do_sample=True,
                         sample_generator=torch.Generator().manual_seed(100 + seed))
        assert set(out.sequences[:, ids.shape[1]:].flatten().tolist()) <= set(model.engine.valid_ids) | {tok.pad_token_id}
        n = min(out.sequences.shape[1], ref.sequences.shape[1])
        agree += int(torch.equal(out.sequences[:, :n], ref.sequences[:, :n]))
        report("generate_do_sample", seed=seed, got=out.sequences[:, ids.shape[1]:].tolist(), want=ref.sequences[:, ids.shape[1]:].tolist())
    assert agree >= 3, agree


def test_lora_assets_change_the_model_like_the_oracle_on_merged_weights(tmp_path):
    """SURVEY 8f-3: `load_lora_assets` (reference lora_loading.py:148-176).  LoRA pairs on LM q_proj/down_proj and on a head FFN
    matrix plus a replaced connector are folded into the packed weights; the closed loop must then match the oracle run on a state
    dict merged independently here (W + (alpha/r) B A in fp32, one rounding to bf16) -- and must differ from the base model."""
    import json
    from safetensors.torch import save_file
    from oracle import vv_oracle as O
    from vibevoice.modular.lora_loading import load_lora_assets
    from vibevoice_b200.modeling import ForcedTokenScript
    model, cfg, tok, sd = make_model("tiny", 1)
    try:
        g = torch.Generator().manual_seed(21)
        rn = lambda *sh: torch.randn(*sh, generator=g)
        targets = {"model.language_model.layers.0.self_attn.q_proj.weight": "base_model.model.layers.0.self_attn.q_proj",
                   "model.language_model.layers.1.mlp.down_proj.weight": "base_model.model.layers.1.mlp.down_proj"}
        head_t = {"model.prediction_head.layers.0.ffn.up_proj.weight": "base_model.model.base.layers.0.ffn.up_proj",
                  "model.prediction_head.layers.1.adaLN_modulation.1.weight": "base_model.model.base.layers.1.adaLN_modulation.1"}
        merged = dict(sd)
        root = tmp_path / "ft" / "lora"
        for d, tg, r, alpha in ((root, targets, 4, 16.0), (root / "diffusion_head", head_t, 2, 4.0)):
            d.mkdir(parents=True, exist_ok=True)
            tens = {}
            for key, mod in tg.items():
                out_f, in_f = sd[key].shape
                A, B = rn(r, in_f) * 0.3, rn(out_f, r) * 0.3
                tens[mod + ".lora_A.weight"], tens[mod + ".lora_B.weight"] = A, B
                merged[key] = (sd[key].float() + (alpha / r) * (B @ A)).to(sd[key].dtype)
            (d / "adapter_config.json").write_text(json.dumps(dict(peft_type="LORA", r=r, lora_alpha=alpha)))
            save_file(tens, str(d / "adapter_model.safetensors"))
        (root / "semantic_connector").mkdir()
        conn = {k.split("semantic_connector.")[1]: (v.float() + 0.05 * rn(*v.shape)).to(v.dtype)
                for k, v in sd.items() if k.startswith("model.semantic_connector.")}
        torch.save(conn, root / "semantic_connector" / "pytorch_model.bin")
        for k, v in conn.items():
            merged["model.semantic_connector." + k] = v

        dc = cfg.decoder_config
        ids = torch.randint(0, dc.vocab_size - 20, (1, 8), generator=g)
        ids[:, -1] = tok.speech_start_id
        script = [_scripted(tok, "ddddx")]
        model.set_ddpm_inference_steps(5)

        def run():
            torch.manual_seed(4)
            return model.generate(input_ids=ids, tokenizer=tok, cfg_scale=1.3, is_prefill=False, logits_processor=[ForcedTokenScript(script)],
                                  max_new_tokens=12, show_progress_bar=False).speech_outputs[0].cpu()
        base_audio = run()
        rep = load_lora_assets(model, str(tmp_path / "ft"))
        assert rep.language_model and rep.diffusion_head_lora and rep.semantic_connector and not rep.acoustic_connector
        tuned = run()
        torch.manual_seed(4)
        ref = O.generate(merged, cfg, ids, None, tok, cfg_scale=1.3, num_steps=5, max_new_tokens=12, forced_tokens=script, kv_bf16=True)
        e, moved = rel_l2(tuned, ref.speech_outputs[0]), rel_l2(tuned, base_audio)
        report("lora_assets", audio_rel_l2=e, moved_from_base=moved)
        assert e < 1e-2 and moved > 10 * e, (e, moved)
    finally:
        if model.engine is not None:
            model.engine.close()


# ---- next-row features (SURVEY 8f): SDE scheduler, refresh_negative=False, streaming-0.5B variant -------------------------------
def test_sde_sampler_vs_oracle():
    """Closed loop with the Gradio demo's scheduler (demo/gradio_demo.py:141-146).  The per-step variance noise is injected on both
    sides (the product would otherwise draw it from the CUDA generator, the oracle from the CPU one)."""
    from oracle import vv_oracle as O
    from vibevoice_b200.modeling import ForcedTokenScript
    model, cfg, tok, sd = make_model("tiny", 2)
    try:
        base = model.model.noise_scheduler
        model.model.noise_scheduler = base.from_config(base.config, algorithm_type="sde-dpmsolver++", beta_schedule="squaredcos_cap_v2")
        model.set_ddpm_inference_steps(5)
        dc = cfg.decoder_config
        g = torch.Generator().manual_seed(5)
        ids = torch.randint(0, dc.vocab_size - 20, (2, 10), generator=g)
        ids[:, -1] = tok.speech_start_id
        scripts = [_scripted(tok, "dddesddx"), _scripted(tok, "ddddddx")]
        pool = torch.randn(64, 5, 4, 64, generator=g)            # [frame][step][2n<=4][64]
        frame = {"i": -1}

        def step_noise_fn(i, n):
            if i == 0:
                frame["i"] += 1
            return pool[frame["i"], i, :2 * n]
        torch.manual_seed(0)
        out = model.generate(input_ids=ids, tokenizer=tok, cfg_scale=1.3, is_prefill=False, logits_processor=[ForcedTokenScript(scripts)],
                             max_new_tokens=20, show_progress_bar=False, _step_noise_fn=step_noise_fn)
        # oracle: same frame noise stream (CPU global RNG), same step noise through sample_speech_tokens' hook
        oframe = {"i": -1}
        orig = O.sample_speech_tokens

        def patched(w, pc, nc, cs, ns, noise, nl=4, eps=1e-5, trace=None, algorithm_type="dpmsolver++", step_noise=None):
            oframe["i"] += 1
            n = pc.shape[0]
            return orig(w, pc, nc, cs, ns, noise, nl, eps, trace, algorithm_type, [pool[oframe["i"], i, :2 * n] for i in range(ns)])
        O.sample_speech_tokens = patched
        try:
            torch.manual_seed(0)
            ref = O.generate(sd, cfg, ids, None, tok, cfg_scale=1.3, num_steps=5, max_new_tokens=20, forced_tokens=scripts, kv_bf16=True,
                             algorithm_type="sde-dpmsolver++")
        finally:
            O.sample_speech_tokens = orig
        assert torch.equal(out.sequences, ref.sequences)
        for r in range(2):
            e = rel_l2(out.speech_outputs[r].cpu(), ref.speech_outputs[r])
            report("sde_generate", row=r, audio_rel_l2=e)
            assert e < 1e-2, (r, e)
        # and the noise term is live: the ODE solver on the same inputs gives different audio
        model.model.noise_scheduler = base
        torch.manual_seed(0)
        ode = model.generate(input_ids=ids, tokenizer=tok, cfg_scale=1.3, is_prefill=False, logits_processor=[ForcedTokenScript(scripts)],
                             max_new_tokens=20, show_progress_bar=False)
        assert rel_l2(ode.speech_outputs[0].cpu(), out.speech_outputs[0].cpu()) > 1e-2
    finally:
        model.engine.close()


def test_refresh_negative_false_vs_oracle():
    """`refresh_negative=False` (reference :503-517), one prompt with two speaker turns: the negative stream keeps every step's input
    and is never restarted."""
    from oracle import vv_oracle as O
    from vibevoice_b200.modeling import ForcedTokenScript
    model, cfg, tok, sd = make_model("tiny", 1)
    try:
        dc = cfg.decoder_config
        g = torch.Generator().manual_seed(31)
        ids = torch.randint(0, dc.vocab_size - 20, (1, 10), generator=g)
        ids[:, -1] = tok.speech_start_id
        script = [_scripted(tok, "ddesdddesdx")]
        model.set_ddpm_inference_steps(5)
        torch.manual_seed(7)
        out = model.generate(input_ids=ids, tokenizer=tok, cfg_scale=1.3, is_prefill=False, logits_processor=[ForcedTokenScript(script)],
                             max_new_tokens=40, show_progress_bar=False, refresh_negative=False)
        torch.manual_seed(7)
        ref = O.generate(sd, cfg, ids, None, tok, cfg_scale=1.3, num_steps=5, max_new_tokens=40, forced_tokens=script, kv_bf16=True,
                         refresh_negative=False)
        torch.manual_seed(7)
        refreshed = O.generate(sd, cfg, ids, None, tok, cfg_scale=1.3, num_steps=5, max_new_tokens=40, forced_tokens=script, kv_bf16=True)
        assert torch.equal(out.sequences, ref.sequences)
        e = rel_l2(out.speech_outputs[0].cpu(), ref.speech_outputs[0])
        moved = rel_l2(ref.speech_outputs[0], refreshed.speech_outputs[0])
        report("refresh_negative_false", audio_rel_l2=e, differs_from_refresh_true=moved)
        assert e < 1e-2 and moved > 10 * e, (e, moved)
        # batched: rows that are not diffusing when another one is get their negative step undone by the reference's mask / cache shift,
        # whose guard hides an OLDER entry and keeps the newest one when the cache holds correct_cnt + 2 entries (:599-624) -- reproduced
        # with vv_kv_delete_slot; speaker turns at different steps in the two rows exercise both outcomes
        m2, _, _, _ = make_model("tiny", 2)
        try:
            ids2 = torch.randint(0, dc.vocab_size - 20, (2, 12), generator=g)
            ids2[:, -1] = tok.speech_start_id
            mask2 = torch.ones(2, 12, dtype=torch.long)
            mask2[1, :3] = 0
            ids2[1, :3] = tok.pad_token_id
            scripts = [_scripted(tok, "ddesdddesddx"), _scripted(tok, "dddddesdddx")]
            m2.set_ddpm_inference_steps(5)
            torch.manual_seed(9)
            out2 = m2.generate(input_ids=ids2, attention_mask=mask2, tokenizer=tok, cfg_scale=1.3, is_prefill=False, max_new_tokens=40,
                               logits_processor=[ForcedTokenScript(scripts)], refresh_negative=False, show_progress_bar=False)
            torch.manual_seed(9)
            ref2 = O.generate(sd, cfg, ids2, mask2, tok, cfg_scale=1.3, num_steps=5, max_new_tokens=40, forced_tokens=scripts, kv_bf16=True,
                              refresh_negative=False)
            assert torch.equal(out2.sequences, ref2.sequences)
            for r in range(2):
                e2 = rel_l2(out2.speech_outputs[r].cpu(), ref2.speech_outputs[r])
                report("refresh_negative_false_batched", row=r, audio_rel_l2=e2)
                assert e2 < 1e-2, (r, e2)
        finally:
            m2.engine.close()
    finally:
        model.engine.close()


def test_streaming_variant_vs_oracle():
    """SURVEY 8f-1 on the GPU: `vibevoice_b200.streaming` (vv_lm_decode_range split stack, row modes, zero-semantic connector) against
    `oracle/vv_streaming.py`, which is pinned to the reference's own streaming generate() (tests/golden/streaming.pt)."""
    from oracle import vv_streaming as VS
    from vibevoice_b200 import streaming as S
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.synth import synth_state_dict
    cfg = preset_config("tiny")
    for eos_bias, n_text, max_new in ((-0.3, 12, 40), (-6.0, 12, 30), (-6.0, 3, 7)):
        sd = VS.streaming_state_dict(synth_state_dict(cfg, 1234, torch.bfloat16), cfg, 1, eos_bias=eos_bias)
        m = S.VibeVoiceStreamingForConditionalGenerationInference(cfg, tts_backbone_num_hidden_layers=1)
        m.load_state_dict(sd)
        try:
            m.set_ddpm_inference_steps(5)
            g = torch.Generator().manual_seed(7)
            prompt = torch.randint(0, 2000, (6,), generator=g)
            text = torch.randint(0, 2000, (n_text,), generator=g)
            torch.manual_seed(0)
            out = m.generate(input_ids=prompt[None], tts_text_ids=text[None], neg_text_input_id=2047, cfg_scale=1.5, max_new_tokens=max_new)
            torch.manual_seed(0)
            ref = VS.generate_streaming(sd, cfg, 1, prompt, text, 2047, cfg_scale=1.5, num_steps=5, max_new_tokens=max_new, kv_bf16=True)
            assert torch.equal(out.sequences, ref.sequences), (out.sequences, ref.sequences)
            assert torch.equal(out.reach_max_step_sample, ref.reach_max_step_sample)
            e = rel_l2(out.speech_outputs[0].cpu(), ref.speech_outputs[0])
            report("streaming_generate", eos_bias=eos_bias, n_text=n_text, audio_rel_l2=e)
            assert e < 1e-2, e
        finally:
            m.engine.close()


def test_streaming_from_pretrained_on_a_checkpoint_directory(tmp_path):
    """`VibeVoiceStreamingForConditionalGenerationInference.from_pretrained(dir, torch_dtype=..., device_map="cuda",
    attn_implementation=...)` as `demo/streaming_inference_from_file.py:244-284` calls it: sharded safetensors with the streaming key names +
    a config.json carrying `tts_backbone_num_hidden_layers`; the loaded model must generate exactly what the in-memory one does."""
    import json
    from safetensors.torch import save_file
    from oracle import vv_streaming as VS
    from vibevoice.modular.modeling_vibevoice_streaming_inference import VibeVoiceStreamingForConditionalGenerationInference as M
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.synth import synth_state_dict
    cfg = preset_config("tiny")
    sd = VS.streaming_state_dict(synth_state_dict(cfg, 1234, torch.bfloat16), cfg, 1, eos_bias=-6.0)
    ck = tmp_path / "VibeVoice-Streaming-synth"
    ck.mkdir()
    d = cfg.to_dict()
    d["model_type"] = "vibevoice_streaming"
    d["tts_backbone_num_hidden_layers"] = 1
    d.pop("semantic_tokenizer_config", None)                  # the streaming config has no semantic tokenizer (configuration_vibevoice_streaming.py:46-52)
    (ck / "config.json").write_text(json.dumps(d))
    keys = sorted(k for k in sd if not k.startswith("model.semantic"))
    half = len(keys) // 2
    for i, part in enumerate((keys[:half], keys[half:])):
        save_file({k: sd[k].contiguous() for k in part}, str(ck / ("model-%05d-of-00002.safetensors" % (i + 1))))
    model = M.from_pretrained(str(ck), torch_dtype=torch.bfloat16, device_map="cuda", attn_implementation="flash_attention_2")
    try:
        model.eval()
        model.set_ddpm_inference_steps(num_steps=5)
        assert model.model.language_model.config._attn_implementation == "flash_attention_2" and model.tts_layers == 1
        g = torch.Generator().manual_seed(7)
        prompt = torch.randint(0, 2000, (6,), generator=g)
        text = torch.randint(0, 2000, (7,), generator=g)
        torch.manual_seed(0)
        out = model.generate(input_ids=prompt[None], tts_text_ids=text[None], neg_text_input_id=2047, cfg_scale=1.5, max_new_tokens=12)
        torch.manual_seed(0)
        ref = VS.generate_streaming(sd, cfg, 1, prompt, text, 2047, cfg_scale=1.5, num_steps=5, max_new_tokens=12, kv_bf16=True)
        assert torch.equal(out.sequences, ref.sequences)
        assert rel_l2(out.speech_outputs[0].cpu(), ref.speech_outputs[0]) < 1e-2
    finally:
        model.engine.close()
    with pytest.raises(Exception):
        M.from_pretrained(str(ck), device_map="cpu")


@pytest.fixture(scope="module")
def real15():
    """VibeVoice-1.5B layer shapes (H=1536, I=8960, 12/2 heads, full-size head and codec), 2 LM layers, small vocab."""
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    cfg = preset_config("1.5b-l2")
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    parts = ("lm", "head", "acoustic_decoder", "semantic", "connectors", "lm_head")
    sd = synth_state_dict(cfg, SEED, torch.bfloat16, parts=parts)
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=1)
    m.load_state_dict(sd, tok)
    yield m, cfg, tok, sd
    m.engine.close()


def test_real_shapes_closed_loop_vs_oracle(real15):
    """Same closed-loop check as the tiny model but at the real 1.5B kernel shapes (K=1536/4608/8960 GEMVs, C up to 2048 codec,
    T up to 3200, tensor-core GEMM and attention paths, 10 diffusion steps)."""
    from oracle import vv_oracle as O
    from vibevoice_b200.modeling import ForcedTokenScript
    model, cfg, tok, sd = real15
    dc = cfg.decoder_config
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(0, dc.vocab_size - 20, (1, 70), generator=g)
    ids[:, -1] = tok.speech_start_id
    script = [_scripted(tok, "ddesdx")]
    model.set_ddpm_inference_steps(10)
    torch.manual_seed(0)
    out = model.generate(input_ids=ids, tokenizer=tok, cfg_scale=1.3, is_prefill=False, logits_processor=[ForcedTokenScript(script)],
                         max_new_tokens=12, show_progress_bar=False)
    torch.manual_seed(0)
    ref = O.generate(sd, cfg, ids, None, tok, cfg_scale=1.3, num_steps=10, max_new_tokens=12, forced_tokens=script, kv_bf16=True)
    assert torch.equal(out.sequences, ref.sequences)
    a, b = out.speech_outputs[0].cpu(), ref.speech_outputs[0]
    assert a.shape == b.shape == (1, 3 * 3200)
    e = rel_l2(a, b)
    report("generate_real_shapes_1.5b", audio_rel_l2=e)
    assert e < 1e-2, e


def test_voice_prompt_and_torch_prefill_vs_oracle():
    """a-9: voice-prompt prefill (acoustic encoder -> Gaussian sample -> connector -> scatter into the prompt) and the PyTorch
    prompt prefill handing K/V to the paged pool, then the usual CUDA loop.  The prefill runs in bf16 on library kernels (like the
    CUDA reference), the oracle in fp32 -> looser audio tolerance (5e-2), token bookkeeping still exact."""
    from oracle import vv_oracle as O
    from vibevoice_b200.modeling import ForcedTokenScript, VibeVoiceForConditionalGenerationInference
    cfg = preset_config("tiny")
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, SEED, torch.bfloat16)
    model = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=1, torch_prefill=True)
    model.load_state_dict(sd, tok)
    g = torch.Generator().manual_seed(8)
    L0 = 30
    ids = torch.randint(0, cfg.decoder_config.vocab_size - 20, (1, L0), generator=g)
    ids[:, -1] = tok.speech_start_id
    sim = torch.zeros(1, L0, dtype=torch.bool)
    sim[0, 5:9] = True
    sim[0, 14:17] = True
    ids[sim] = tok.speech_diffusion_id
    wavs = torch.zeros(2, 3200 * 3 + 100)
    wavs[0] = torch.randn(wavs.shape[1], generator=g) * 0.05
    wavs[1, :3200 * 2 + 7] = torch.randn(3200 * 2 + 7, generator=g) * 0.05
    masks = torch.zeros(2, 4, dtype=torch.bool)
    masks[0, :4] = True
    masks[1, :3] = True
    noise = (torch.randn(2, generator=g), torch.randn(2, 4, 64, generator=g))
    want_emb = O.voice_prompt_embeds(sd, cfg, wavs, masks, noise=noise)
    got_emb = model._voice(wavs, masks, float(sd["model.speech_scaling_factor"]), float(sd["model.speech_bias_factor"]), noise=noise).cpu()
    e = rel_l2(got_emb, want_emb)
    report("voice_prompt_embeds", rel_l2=e)
    assert e < 1e-4, e
    script = [_scripted(tok, "dddx")]
    model.set_ddpm_inference_steps(5)
    torch.manual_seed(0)
    out = model.generate(input_ids=ids, tokenizer=tok, cfg_scale=1.3, is_prefill=True, speech_tensors=wavs, speech_masks=masks,
                         speech_input_mask=sim, _voice_noise=noise, logits_processor=[ForcedTokenScript(script)], max_new_tokens=8,
                         show_progress_bar=False)
    torch.manual_seed(0)
    ref = O.generate(sd, cfg, ids, None, tok, cfg_scale=1.3, num_steps=5, max_new_tokens=8, forced_tokens=script, kv_bf16=True,
                     speech_embeds=[(sim[0], want_emb)])
    assert torch.equal(out.sequences, ref.sequences)
    a, b = out.speech_outputs[0].cpu(), ref.speech_outputs[0]
    assert a.shape == b.shape == (1, 9600)
    e = rel_l2(a, b)
    report("generate_voice_prompt_torch_prefill", audio_rel_l2=e)
    assert e < 5e-2, e
    model.engine.close()


def test_wgmma_gemm_forced_everywhere():
    """gemm_wgmma_kernel (warpgroup wgmma.mma_async, register accumulators) is selected automatically only for wide GEMMs; force it for
    EVERY M > 8 GEMM (VV_WGMMA=2) and re-check the GEMM-vs-torch cases and a closed codec loop through the tensor-core path."""
    import ctypes as C
    old = os.environ.get("VV_WGMMA")
    os.environ["VV_WGMMA"] = "2"
    try:
        m, cfg, tok, sd = make_model("tiny", 1)
    finally:
        if old is None:
            os.environ.pop("VV_WGMMA", None)
        else:
            os.environ["VV_WGMMA"] = old
    eng = m.engine
    P = lambda t: C.c_void_p(t.data_ptr())
    for (M, N, K) in [(40, 2048, 512), (200, 1024, 256), (70, 96, 40), (60, 21504, 1536), (130, 200, 72)]:
        g = torch.Generator().manual_seed(M + N + K)
        W = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
        x, bias = torch.randn(M, K, generator=g), torch.randn(N, generator=g) * 0.1
        Wd, xd, bd = W.cuda(), x.cuda(), bias.cuda()
        torch.cuda.synchronize()
        for epi in (NV.EPI_NONE, NV.EPI_GELU, NV.EPI_RESID):
            y = torch.full((M, N), 0.25, device="cuda")
            torch.cuda.synchronize()
            with torch.cuda.stream(eng.stream):
                NV.check(eng.lib.vv_debug_gemv(eng.h, P(Wd), P(bd), P(xd), P(y), M, N, K, NV.PRO_NONE, None, 1e-5, epi, eng.s))
            eng.sync()
            ref = x @ W.float().T + bias
            ref = torch.nn.functional.gelu(ref) if epi == NV.EPI_GELU else (ref + 0.25 if epi == NV.EPI_RESID else ref)
            e = rel_l2(y, ref)
            report("wgmma_gemm", M=M, N=N, K=K, epi=epi, rel_l2=e)
            assert e < 2e-5, (M, N, K, epi, e)
    from oracle import vv_oracle as O
    eng.codec_state_reset()
    a, s_ = O.StreamState(1), O.StreamState(1)
    g = torch.Generator().manual_seed(5)
    scale, bias_f = float(sd["model.speech_scaling_factor"]), float(sd["model.speech_bias_factor"])
    for f in range(3):
        lat = torch.randn(1, 64, generator=g)
        with torch.cuda.stream(eng.stream):
            eng.latent.copy_(lat.cuda())
        eng.upload_frame_inputs(torch.zeros(1, 64), [0])
        eng.codec_decode(); eng.semantic_encode(); eng.sync()
        audio = O.decoder_frame(sd, cfg.acoustic_tokenizer_config, (lat / scale - bias_f)[:, None, :], a, [0])
        sem = O.encoder_frame(sd, cfg.semantic_tokenizer_config, audio, s_, [0])
        assert rel_l2(eng.audio.cpu(), audio[:, 0]) < 2e-3 and rel_l2(eng.feat.cpu(), sem[:, 0]) < 2e-3
    eng.close()
