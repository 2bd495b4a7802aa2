"""`-m gpu`: the streaming-0.5B request queue (`serving.StreamingRequestQueue`) and the two kernels it batches.

  * `Engine.eos_probs`: every row bit-equal to `vv_eos_prob` on that row alone, at n = 1..8 rows in shuffled order, and within the float64
    bound of `test_gpu_streaming_demo.py::test_eos_prob_kernel_vs_float64`;
  * `Engine.tts_type_embed_rows`: bit-equal to the fp32 add, with sources that are also destinations;
  * solo `generate()` on a four-slot model (slot 0) against the streaming oracle, at the bounds of `test_generate_from_preset_vs_oracle`;
  * the queue against solo `generate()` runs of the same requests at max_slots 2 and 4, on tiny, streaming-0.5b-l4 and the shipped
    geometry from the preset fixture, with EOS biases +20 / -20 (decisions with a clear margin): sequences and flags identical, audio
    rel-L2 < 1e-2, streamer chunks equal to the returned audio; and every tick makes at most one lower-stack and one upper-stack launch.
"""
import copy
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

from vibevoice_b200.configuration import preset_config
from vibevoice_b200.streamer import AudioStreamer
from vibevoice_b200.synth import synth_state_dict

from test_gpu_parity import SEED, rel_l2, report
from test_gpu_streaming_demo import PARTS, TTS_LAYERS, _cfg, _cut_lengths, _preset


def _model(cfg, sd, tts, slots):
    from vibevoice_b200 import streaming as S
    m = S.VibeVoiceStreamingForConditionalGenerationInference(cfg, tts_backbone_num_hidden_layers=tts, max_slots=slots)
    m.load_state_dict(sd)
    return m


def _checkpoint(preset, eos_bias=-0.3, dtype=torch.float32):
    from oracle import vv_streaming as VS
    if preset == "shipped":
        cfg, tts = _cfg(), TTS_LAYERS
    else:
        cfg, tts = preset_config(preset), (1 if preset == "tiny" else 3)
    base = synth_state_dict(cfg, SEED, dtype, parts=PARTS)
    return cfg, VS.streaming_state_dict(base, cfg, tts, eos_bias=eos_bias), tts


@pytest.mark.parametrize("preset", ["tiny", "streaming-0.5b-l4"])
def test_eos_probs_rows_are_the_single_row_kernel(preset):
    cfg, sd, tts = _checkpoint(preset)
    m = _model(cfg, sd, tts, 4)
    eng = m.engine
    try:
        H = cfg.decoder_config.hidden_size
        w1, b1 = sd["tts_eos_classifier.fc1.weight"].double(), sd["tts_eos_classifier.fc1.bias"].double()
        w2, b2 = sd["tts_eos_classifier.fc2.weight"].double()[0], sd["tts_eos_classifier.fc2.bias"].double()[0]
        g = torch.Generator().manual_seed(3)
        rnd = random.Random(3)
        for scale in (1.0, 1e3):
            hid = torch.randn(2 * eng.B, H, generator=g) * scale
            with torch.cuda.stream(eng.stream):
                eng.hidden.copy_(hid.to(eng.device))
            single = []
            for r in range(2 * eng.B):
                single.append((eng.eos_prob(eng.hidden[r]), eng.eos_logit))
            for r, (p, lg) in enumerate(single):
                pre = w1 @ hid[r].double() + b1
                ref = float(w2 @ torch.relu(pre) + b2)
                mag = float(w2.abs() @ ((w1 * hid[r].double()).abs().sum(1) + b1.abs()) + b2.abs())
                assert abs(lg - ref) <= 1e-6 * mag, (scale, r, lg, ref, mag)
            for n in range(1, 9):
                for _ in range(3):
                    rows = rnd.sample(range(2 * eng.B), n)
                    probs = eng.eos_probs(rows)
                    assert probs == [single[r][0] for r in rows], (n, rows)
                    assert eng.eos_logits == [single[r][1] for r in rows], (n, rows)
            report("eos_probs_rows", preset=preset, scale=scale)
        with pytest.raises(ValueError):
            eng.eos_probs(list(range(9)))
    finally:
        eng.close()


def test_tts_type_embed_rows_is_the_fp32_add():
    cfg, sd, tts = _checkpoint("streaming-0.5b-l4")
    m = _model(cfg, sd, tts, 4)
    eng = m.engine
    try:
        H = cfg.decoder_config.hidden_size
        types = sd["model.tts_input_types.weight"].float()
        g = torch.Generator().manual_seed(9)
        src = torch.randn(6, H, generator=g) * 3
        src_rows, type_ids, dst_rows = [0, 5, 2, 2, 3, 1, 4, 0, 5, 1, 3, 2, 0, 4, 1, 5], [1, 0, 0, 1] * 4, list(range(16))
        dst = torch.full((16, H), float("nan"), device=eng.device)
        s_dev = src.to(eng.device)
        torch.cuda.synchronize()                                         # the engine reads its inputs on its own stream
        eng.tts_type_embed_rows(s_dev, src_rows, type_ids, dst_rows, dst)
        eng.sync()
        for i in range(16):
            assert torch.equal(dst[i].cpu(), src[src_rows[i]] + types[type_ids[i]]), i
        # in place, with sources that are destinations: rows 0 and 1 swap (each reads the other), row 2 reads itself, row 3 reads row 0
        buf = src[:4].clone().to(eng.device)
        torch.cuda.synchronize()
        eng.tts_type_embed_rows(buf, [1, 0, 2, 0], [1, 0, 1, 0], [0, 1, 2, 3], buf)
        eng.sync()
        want = torch.stack([src[1] + types[1], src[0] + types[0], src[2] + types[1], src[0] + types[0]])
        assert torch.equal(buf.cpu(), want)
        with pytest.raises(ValueError):
            eng.tts_type_embed_rows(buf, [4], [0], [0], buf)
    finally:
        eng.close()


@pytest.mark.parametrize("case,eos_bias,n_text,max_new,cfg_scale", [("eos", 20.0, 12, 40, 1.5), ("windows", -20.0, 12, 30, 1.5),
                                                                    ("short", -20.0, 3, 7, 1.3)])
def test_solo_generate_on_four_slot_model_vs_oracle(case, eos_bias, n_text, max_new, cfg_scale):
    from streaming_oracle import generate_from_prefilled
    cfg, sd, tts = _checkpoint("shipped", eos_bias, torch.bfloat16)
    preset, lengths = _preset(), _cut_lengths()
    g = torch.Generator().manual_seed(11)
    text = torch.randint(0, 2000, (n_text,), generator=g)
    tts_ids = torch.full((lengths["tts_lm"],), 3, dtype=torch.long)
    m = _model(cfg, sd, tts, 4)
    try:
        m.set_ddpm_inference_steps(5)
        torch.manual_seed(0)
        out = m.generate(input_ids=torch.full((1, lengths["lm"]), 3), tts_lm_input_ids=tts_ids[None], tts_text_ids=text[None], neg_text_input_id=3,
                         cfg_scale=cfg_scale, max_new_tokens=max_new, all_prefilled_outputs=copy.deepcopy(preset))
    finally:
        m.engine.close()
    torch.manual_seed(0)
    ref = generate_from_prefilled(sd, cfg, tts, preset, tts_ids, text, cfg_scale=cfg_scale, num_steps=5, max_new_tokens=max_new, kv_bf16=True)
    assert torch.equal(out.sequences, ref.sequences), (out.sequences, ref.sequences)
    assert torch.equal(out.reach_max_step_sample, ref.reach_max_step_sample)
    e = rel_l2(out.speech_outputs[0].cpu(), ref.speech_outputs[0])
    report("streaming_generate_four_slots", case=case, audio_rel_l2=e)
    assert e < 1e-2, e


def _requests(preset, n, seed):
    """n requests: text lengths 0, < 5 and several windows; steps 3 / 5 / 8, CFG 1.0 / 1.3 / 1.5 and length limits up to 40 new tokens
    mixed; at the shipped geometry every other request starts from the preset fixture, the rest (and every request elsewhere) from
    input_ids.  CFG and length stay within the bounds of `test_generate_from_preset_vs_oracle`: beyond them the closed loop amplifies
    the stream kernel's non-reproducible fp32 atomics (at CFG 3.0, 29 text-less frames from the preset differ by 0.15 rel-L2 between two
    solo runs of the same program on the H100), and the 1e-2 bound would measure that, not the queue."""
    rnd = random.Random(seed)
    g = torch.Generator().manual_seed(seed)
    lengths = _cut_lengths() if preset == "shipped" else None
    reqs = []
    for i in range(n):
        n_text = [3, 0, 12, 1, 23, 7][i % 6]
        r = dict(text=torch.randint(0, 2000, (n_text,), generator=g), cfg_scale=rnd.choice([1.0, 1.3, 1.5]), steps=rnd.choice([3, 5, 8]),
                 max_new_tokens=rnd.randint(6, 40), seed=rnd.randint(0, 10 ** 6), streamer=i % 2 == 1)
        if lengths is not None and i % 2 == 0:
            r["kw"] = dict(input_ids=torch.full((1, lengths["lm"]), 3), tts_lm_input_ids=torch.full((1, lengths["tts_lm"]), 3), neg_text_input_id=3)
            r["preset"] = True
        else:
            r["kw"] = dict(input_ids=torch.randint(0, 2000, (rnd.randint(2, 9),), generator=g)[None], neg_text_input_id=2047)
            r["preset"] = False
        reqs.append(r)
    return reqs


def _kw(r, preset):
    kw = dict(r["kw"])
    if r["preset"]:
        kw["all_prefilled_outputs"] = copy.deepcopy(preset)
    return kw


@pytest.mark.parametrize("preset", ["tiny", "streaming-0.5b-l4", "shipped"])
@pytest.mark.parametrize("eos_bias", [20.0, -20.0])
def test_queue_matches_solo_runs(preset, eos_bias):
    from vibevoice_b200 import serving
    cfg, sd, tts = _checkpoint(preset, eos_bias, torch.bfloat16)
    pre = _preset() if preset == "shipped" else None
    reqs = _requests(preset, 7, 5)
    for slots in (2, 4):
        m = _model(cfg, sd, tts, slots)
        eng = m.engine
        try:
            eng.kv_init(16384)
            refs = []
            for r in reqs:
                torch.manual_seed(r["seed"])
                m.set_ddpm_inference_steps(r["steps"])
                refs.append(m.generate(tts_text_ids=r["text"][None], cfg_scale=r["cfg_scale"], max_new_tokens=r["max_new_tokens"], **_kw(r, pre)))
            q = serving.StreamingRequestQueue(m, max_total_tokens=16384)
            streams, rids = {}, []
            for r in reqs:
                st = AudioStreamer(1) if r["streamer"] else None
                rid = q.submit(tts_text_ids=r["text"], cfg_scale=r["cfg_scale"], steps=r["steps"], max_new_tokens=r["max_new_tokens"],
                               seed=r["seed"], audio_streamer=st, **_kw(r, pre))
                rids.append(rid)
                streams[rid] = st
            calls = []
            inner = eng.lm_decode_range

            def logged(begin, end, final_norm, out=None):
                calls.append(begin)
                return inner(begin, end, final_norm, out)
            eng.lm_decode_range = logged
            outs, worst = {}, 0.0
            while len(outs) < len(reqs):
                calls.clear()
                for rid, out in q.step():
                    outs[rid] = out
                assert calls.count(0) <= 1 and len(calls) - calls.count(0) <= 1, calls   # one lower-, one upper-stack program per tick
            del eng.lm_decode_range
            for rid, r, ref in zip(rids, reqs, refs):
                out = outs[rid]
                assert torch.equal(out.sequences, ref.sequences), (slots, out.sequences, ref.sequences)
                assert torch.equal(out.reach_max_step_sample, ref.reach_max_step_sample)
                a, b = out.speech_outputs[0], ref.speech_outputs[0]
                assert (a is None) == (b is None)
                if a is not None:
                    assert a.shape == b.shape
                    e = rel_l2(a.cpu(), b.cpu())
                    worst = max(worst, e)
                    assert e < 1e-2, (slots, e)
                st = streams[rid]
                if st is not None:
                    ch = list(st.get_stream(0))
                    got = torch.cat(ch, dim=-1) if ch else None
                    assert (got is None) == (a is None) and (a is None or torch.equal(got, a.cpu()))
            assert q._pages_used == 0
            ends = sum(bool(o.reach_max_step_sample[0]) for o in outs.values())
            report("streaming_queue_vs_solo", preset=preset, eos_bias=eos_bias, slots=slots, audio_rel_l2_max=worst, ended_by_limit=ends)
        finally:
            eng.close()
