"""`-m gpu` tests of the native prompt prefill (`vv_lm_prefill`, csrc/vv_prefill.cuh): K/V of every layer and the last hidden state against
`oracle.qwen2_forward(act_bf16=True)` with a bf16 cache, compared with the error the PyTorch prefill (`TorchPrefill`, bf16 library
kernels) makes on the same inputs; continuation, workspace independence and error codes; a 61 440-token prompt; and `generate()`."""
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
CAP = 1e-2                     # absolute cap on every rel-L2 against the oracle (K, V per layer, last hidden state)
OUT = os.environ.get("VV_REPORT_DIR") or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "reports")
LENS = [1, 63, 64, 65, 200, 1000]
PARTS = ("lm", "head", "acoustic_decoder", "semantic", "connectors", "lm_head")     # all but the optional acoustic encoder
PRESETS = ["tiny", "small", "tiny64", "1.5b-l2", "7b-l2", "streaming-0.5b-l4"]


def rel_l2(a, b) -> float:
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def report(name, **kv):
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "parity_report.jsonl"), "a") as f:
        f.write(json.dumps(dict(test=name, **kv)) + "\n")


def make_model(preset, max_batch=1, prefill_impl=None, parts=None):
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    cfg = preset_config(preset)
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, SEED, torch.bfloat16) if parts is None else synth_state_dict(cfg, SEED, torch.bfloat16, parts=parts)
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=max_batch, prefill_impl=prefill_impl)
    m.load_state_dict(sd, tok)
    return m, cfg, tok, sd


def _embeds(cfg, L, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(L, cfg.decoder_config.hidden_size, generator=g) * 0.5


def _native(eng, seq, e, pos0=0, ws=None):
    h = eng.lm_prefill(seq, e.cuda(), pos0=pos0, workspace_bytes=ws)
    eng.sync()
    return h.cpu()


def _kv(eng, seq, L):
    dc = eng.config.decoder_config
    return [tuple(t.float().cpu() for t in eng.kv_read(seq, l, 0, L)) for l in range(dc.num_hidden_layers)]


@pytest.mark.parametrize("preset", PRESETS)
def test_prefill_parity_vs_oracle_and_torch_prefill(preset):
    """Every layer's K/V (read back from the pool) and the last hidden state at L in {1, 63, 64, 65, 200, 1000} (+ 5000 at 1.5b-l2): the
    native error against the oracle is no larger than TorchPrefill's on the same weights and inputs, and below CAP."""
    from oracle import vv_oracle as O
    from vibevoice_b200.prefill import TorchPrefill
    m, cfg, tok, sd = make_model(preset, parts=PARTS)
    eng = m.engine
    try:
        dc = cfg.decoder_config
        lens = LENS + ([5000] if preset == "1.5b-l2" else [])
        Lmax = max(lens)
        eng.kv_init(2 * Lmax + 256)
        e = _embeds(cfg, Lmax, 7)
        sd32 = {k: v.float() for k, v in sd.items() if k.startswith("model.language_model.")}
        cache = O.KVCache(dc.num_hidden_layers, kv_bf16=True)
        want_h = O.qwen2_forward(sd32, dc, e, cache, 0, act_bf16=True)          # causal: row L-1 / the first L keys are the prefix-L answer
        tp = TorchPrefill(cfg, sd32, eng.device)
        for L in lens:
            got_h = _native(eng, 0, e[:L])
            with torch.cuda.stream(eng.stream):
                tor_h = tp.run(eng, 1, e[:L].cuda())
            eng.sync()
            tor_h = tor_h.float().cpu()
            nat_kv, tor_kv = _kv(eng, 0, L), _kv(eng, 1, L)
            rows = []
            for l in range(dc.num_hidden_layers):
                wk, wv = cache.k[l][:, :L].transpose(0, 1), cache.v[l][:, :L].transpose(0, 1)
                rows.append(dict(layer=l, k=rel_l2(nat_kv[l][0], wk), v=rel_l2(nat_kv[l][1], wv),
                                 k_torch=rel_l2(tor_kv[l][0], wk), v_torch=rel_l2(tor_kv[l][1], wv)))
            eh, eh_t = rel_l2(got_h, want_h[L - 1]), rel_l2(tor_h, want_h[L - 1])
            report("prefill_parity", preset=preset, L=L, hidden=eh, hidden_torch=eh_t, layers=rows)
            assert eh <= max(eh_t, 1e-6) and eh < CAP, (preset, L, eh, eh_t)
            for r in rows:
                assert r["k"] <= max(r["k_torch"], 1e-6) and r["v"] <= max(r["v_torch"], 1e-6), (preset, L, r)
                assert r["k"] < CAP and r["v"] < CAP, (preset, L, r)
            eng.kv_set_len(0, 0)
            eng.kv_set_len(1, 0)
    finally:
        eng.close()


@pytest.mark.parametrize("preset,L,a", [("tiny", 200, 77), ("tiny64", 1000, 333), ("1.5b-l2", 1000, 130)])
def test_prefill_continuation(preset, L, a):
    """[0, a) then [a, L) with a not a multiple of 64 gives the same K/V and last hidden state as one call over [0, L) -- bit for bit, since
    no row's arithmetic depends on the rows it is chunked with -- and so the same error against the oracle (below CAP)."""
    from oracle import vv_oracle as O
    m, cfg, tok, sd = make_model(preset, parts=PARTS)
    eng = m.engine
    try:
        dc = cfg.decoder_config
        eng.kv_init(2 * L + 256)
        e = _embeds(cfg, L, 11)
        h_one = _native(eng, 0, e)
        _native(eng, 1, e[:a])
        eng.kv_set_len(1, a)
        h_two = _native(eng, 1, e[a:], pos0=a)
        kv1, kv2 = _kv(eng, 0, L), _kv(eng, 1, L)
        cache = O.KVCache(dc.num_hidden_layers, kv_bf16=True)
        want = O.qwen2_forward({k: v.float() for k, v in sd.items() if k.startswith("model.language_model.")}, dc, e, cache, 0, act_bf16=True)[-1]
        e1, e2 = rel_l2(h_one, want), rel_l2(h_two, want)
        report("prefill_continuation", preset=preset, L=L, a=a, hidden_one=e1, hidden_two=e2)
        assert e2 < CAP and e1 < CAP
        assert torch.equal(h_one, h_two)
        for l in range(dc.num_hidden_layers):
            assert torch.equal(kv1[l][0], kv2[l][0]) and torch.equal(kv1[l][1], kv2[l][1]), l
    finally:
        eng.close()


def test_prefill_workspace_and_errors():
    """Minimum and large workspace: bit-identical K/V and hidden state.  One byte below the minimum: VV_ERR_INVALID and no launch.  Pool
    too small: VV_ERR_NOMEM.  Bad seq / n / pos0: VV_ERR_INVALID.  Before vv_finalize_weights or vv_kv_init: VV_ERR_STATE."""
    from vibevoice_b200.engine import Engine
    m, cfg, tok, sd = make_model("1.5b-l2", parts=PARTS)
    eng = m.engine
    P = lambda t: C.c_void_p(t.data_ptr())
    try:
        dc = cfg.decoder_config
        L, H = 1000, dc.hidden_size
        e = _embeds(cfg, L, 3).cuda()
        out = torch.empty(H, device="cuda")
        rc = eng.lib.vv_lm_prefill(eng.h, 0, 0, L, P(e), P(out), P(torch.empty(64 << 20, dtype=torch.uint8, device="cuda")), 64 << 20, eng.s)
        assert rc == -3                                                          # no KV pool yet
        eng.kv_init(4 * L)
        need = eng.lm_prefill_workspace_bytes(L)
        h_min = _native(eng, 0, e, ws=need)
        kv_min = _kv(eng, 0, L)
        h_big = _native(eng, 1, e, ws=need * 64)
        kv_big = _kv(eng, 1, L)
        assert torch.equal(h_min, h_big)
        for a, b in zip(kv_min, kv_big):
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        work = torch.empty(need, dtype=torch.uint8, device="cuda")
        n0 = eng.launch_count()
        assert eng.lib.vv_lm_prefill(eng.h, 0, 0, L, P(e), P(out), P(work), need - 1, eng.s) == -1
        assert eng.launch_count() == n0
        for seq, pos0, n in ((-1, 0, L), (2, 0, L), (0, 0, 0), (0, -1, L), (0, dc.max_position_embeddings - 10, 11)):
            assert eng.lib.vv_lm_prefill(eng.h, seq, pos0, n, P(e), P(out), P(work), need, eng.s) == -1, (seq, pos0, n)
        assert eng.launch_count() == n0
        eng.kv_set_len(0, 0)
        eng.kv_set_len(1, 0)
        big = eng.kv_pages * 64 + 64
        e_big = torch.zeros(big, H, device="cuda")
        assert eng.lib.vv_lm_prefill(eng.h, 0, 0, big, P(e_big), P(out), P(work), need, eng.s) == -4
        bare = Engine(cfg, m._valid_ids(tok), 1)
        try:
            assert bare.lib.vv_lm_prefill(bare.h, 0, 0, L, P(e), P(out), P(work), need, bare.s) == -3
            assert bare.lib.vv_lm_prefill_workspace(bare.h, L) == -3
        finally:
            bare.close()
    finally:
        eng.close()


def test_prefill_long_context():
    """61 440 tokens on 1.5b-l2: layer-0 K/V at every position against an fp32 CPU computation; the last hidden state against TorchPrefill;
    4 decode steps after each prefill against the oracle over that prefill's own bf16 pool contents (2e-3, as for long-context decode)."""
    from oracle import vv_oracle as O
    from vibevoice_b200.prefill import TorchPrefill
    m, cfg, tok, sd = make_model("1.5b-l2", parts=PARTS)
    eng = m.engine
    try:
        dc = cfg.decoder_config
        L, nl, nkv, hd = 61440, dc.num_hidden_layers, dc.num_key_value_heads, dc.head_dim
        sd32 = {k: v.float() for k, v in sd.items() if k.startswith("model.language_model.")}
        eng.kv_init(L + 512)
        e = _embeds(cfg, L, 5)
        results = {}
        for impl in ("native", "torch"):
            eng.kv_set_len(0, 0)
            eng.kv_set_len(1, 0)
            if impl == "native":
                h = _native(eng, 0, e)
            else:
                tp = TorchPrefill(cfg, sd32, eng.device)
                with torch.cuda.stream(eng.stream):
                    h = tp.run(eng, 0, e.cuda())
                eng.sync()
                h = h.float().cpu()
                del tp
                torch.cuda.empty_cache()
            eng.kv_set_len(0, L)
            kv = [eng.kv_read(0, l, 0, L) for l in range(nl)]
            if impl == "native":                                   # layer 0 depends on the embeddings only
                p = "model.language_model.layers.0"
                x = O.round_bf16(O.rms_norm(e, sd32[f"{p}.input_layernorm.weight"], dc.rms_norm_eps))
                k = (x @ sd32[f"{p}.self_attn.k_proj.weight"].T + sd32[f"{p}.self_attn.k_proj.bias"]).view(L, nkv, hd).transpose(0, 1)
                v = (x @ sd32[f"{p}.self_attn.v_proj.weight"].T + sd32[f"{p}.self_attn.v_proj.bias"]).view(L, nkv, hd)
                k = O._rope(k, torch.arange(L), dc.rope_theta).transpose(0, 1)
                gk, gv = kv[0][0].float().cpu(), kv[0][1].float().cpu()
                ek = ((gk - k).flatten(1).norm(dim=1) / k.flatten(1).norm(dim=1)).max().item()
                ev = ((gv - v).flatten(1).norm(dim=1) / v.flatten(1).norm(dim=1)).max().item()
                report("prefill_long_layer0", L=L, k_max_row_rel_l2=ek, v_max_row_rel_l2=ev)
                assert ek < 5e-3 and ev < 5e-3, (ek, ev)
            cache = O.KVCache(nl, kv_bf16=True)
            for l in range(nl):
                cache.preload(l, kv[l][0].float().cpu().transpose(0, 1).contiguous(), kv[l][1].float().cpu().transpose(0, 1).contiguous())
            del kv
            g = torch.Generator().manual_seed(17)
            errs = []
            for step in range(4):
                xin = torch.randn(2, dc.hidden_size, generator=g) * 0.05
                with torch.cuda.stream(eng.stream):
                    eng.embeds.copy_(xin.cuda())
                eng.lm_decode()
                eng.read_tokens()
                want = O.qwen2_forward(sd, dc, xin[0][None], cache, len(cache))[0]
                eng.kv_commit([1, 0])
                errs.append(rel_l2(eng.hidden[0].cpu(), want))
            report("prefill_long_decode", impl=impl, L=L, rel_l2=errs)
            assert max(errs) < 2e-3, (impl, errs)
            results[impl] = h
        e_h = rel_l2(results["native"], results["torch"])
        report("prefill_long_hidden_vs_torch", L=L, rel_l2=e_h)
        assert e_h < 5e-2, e_h
    finally:
        eng.close()


def _scripted(tok, plan):
    d = dict(d=tok.speech_diffusion_id, e=tok.speech_end_id, s=tok.speech_start_id, x=tok.eos_token_id)
    return [d[c] for c in plan]


@pytest.mark.parametrize("preset", ["tiny", "1.5b-l2"])
def test_generate_native_prefill(preset):
    """`generate(prefill_impl="native")` on a model built with `prefill_impl="native"` (no TorchPrefill, no bf16 LM copy): B = 1 and B = 2
    ragged left-padded, with and without voice prompts.  Tokens equal to `oracle.generate`, audio within 5e-2 (the TorchPrefill test's
    bound).  The first prefill call grows device memory by less than 64 MB beyond its workspace."""
    from oracle import vv_oracle as O
    from vibevoice_b200.modeling import ForcedTokenScript
    m, cfg, tok, sd = make_model(preset, max_batch=2, prefill_impl="native")
    eng = m.engine
    try:
        assert m._prefill is None and not m._lm_sd
        dc = cfg.decoder_config
        eng.kv_init(8192)
        e = _embeds(cfg, 4096, 1).cuda()
        ws = eng.lm_prefill_workspace_bytes(4096) * 64
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0 = torch.cuda.mem_get_info()[0]
        eng.lm_prefill(0, e, workspace_bytes=ws)
        torch.cuda.synchronize()
        grow = free0 - torch.cuda.mem_get_info()[0] - ws
        report("prefill_memory_growth", preset=preset, workspace=ws, growth_beyond_workspace=grow)
        assert grow < 64 << 20, grow
        del e
        g = torch.Generator().manual_seed(9)
        T, F = 3 * 3200 + 100, 4
        wavs = torch.randn(3, T, generator=g) * 0.05
        wavs[1, 2 * 3200 + 7:] = 0
        vmask = torch.zeros(3, F, dtype=torch.bool)
        vmask[0, :4] = True
        vmask[1, :3] = True
        vmask[2, :2] = True
        noise = (torch.randn(3, generator=g), torch.randn(3, F, 64, generator=g))
        sdf = {k: v.float() for k, v in sd.items()}
        want_emb = O.voice_prompt_embeds(sdf, cfg, wavs, vmask, noise=noise)
        L0 = 24
        for voice in (False, True):
            for B in (1, 2):
                ids = torch.randint(0, dc.vocab_size - 20, (B, L0), generator=g)
                ids[:, -1] = tok.speech_start_id
                mask = torch.ones(B, L0, dtype=torch.long)
                sim = torch.zeros(B, L0, dtype=torch.bool)
                if B == 2:
                    mask[1, :5] = 0
                    ids[1, :5] = tok.pad_token_id
                extra, speech = {}, None
                if voice:
                    nv = 1 if B == 1 else 3
                    sim[0, 3:7] = True
                    if B == 2:
                        sim[1, 7:10] = True
                        sim[1, 13:15] = True
                    ids[sim] = tok.speech_diffusion_id
                    counts = sim.sum(-1).tolist()
                    offs = [0, counts[0], counts[0] + (counts[1] if B == 2 else 0)]
                    emb = want_emb[: offs[B]]
                    speech = [(sim[r][mask[r].bool()], emb[offs[r]:offs[r + 1]]) for r in range(B)]
                    extra = dict(speech_tensors=wavs[:nv], speech_masks=vmask[:nv], speech_input_mask=sim, _voice_noise=(noise[0][:nv], noise[1][:nv]))
                scripts = [_scripted(tok, "dddx"), _scripted(tok, "ddesdx")][:B]
                m.set_ddpm_inference_steps(5)
                torch.manual_seed(0)
                out = m.generate(input_ids=ids, attention_mask=mask, tokenizer=tok, cfg_scale=1.3, is_prefill=voice,
                                 logits_processor=[ForcedTokenScript(scripts)], max_new_tokens=12, show_progress_bar=False,
                                 prefill_impl="native", **extra)
                torch.manual_seed(0)
                ref = O.generate(sdf, cfg, ids, mask, tok, cfg_scale=1.3, num_steps=5, max_new_tokens=12, forced_tokens=scripts, kv_bf16=True,
                                 speech_embeds=speech)
                assert torch.equal(out.sequences, ref.sequences), (voice, B)
                assert torch.equal(out.reach_max_step_sample, ref.reach_max_step_sample)
                for r in range(B):
                    a, b = out.speech_outputs[r].cpu(), ref.speech_outputs[r]
                    assert a.shape == b.shape
                    err = rel_l2(a, b)
                    report("generate_native_prefill", preset=preset, voice=voice, B=B, row=r, audio_rel_l2=err)
                    assert err < 5e-2, (voice, B, r, err)
    finally:
        eng.close()
