"""`-m gpu` tests of request priorities: parked KV sequences (`vv_kv_park*`), one row's codec state saved and loaded (`vv_codec_state_*`),
and `RequestQueue` preempting lower-priority rows, with every request still equal to its solo `generate()`."""
import pytest
import torch

from test_gpu_queue import requests as plain_requests
from test_gpu_voice_preset import (PARTS, assert_same, embeds, full_request, kv_all, make_model, prefix_inputs, refused, same_kv,
                                   solo_preset)

pytestmark = pytest.mark.gpu


def refused_quietly(eng, fn):
    """refused with an error message and no launch"""
    n = eng.launch_count()
    refused(fn)
    assert eng.launch_count() == n and eng.lib.vv_last_error()


def test_park_runtime():
    m, cfg, tok = make_model("tiny", 3, parts=PARTS, prefill_impl="native")
    eng = m.engine
    try:
        B, dc = eng.B, cfg.decoder_config
        eng.kv_init(4096)
        total = eng.kv_pages
        e = embeds(cfg, 200, 1)
        eng.lm_prefill(0, e)
        eng.kv_set_len(0, 200)
        src = kv_all(eng, 0, 0, 200)
        eng.lm_prefill(1, embeds(cfg, 10, 2))
        eng.kv_set_len(1, 10)
        eng.sync()
        free0, n0 = eng.kv_pages_free(), eng.launch_count()
        h = eng.kv_park(0)
        assert eng.launch_count() == n0                                   # parking launches nothing
        assert eng.kv_len(0) == 0 and eng.kv_seq_pages(0) == 0 and eng.kv_parked_pages(h) == 4
        assert eng.kv_pages_free() == free0                               # parked pages stay used
        refused_quietly(eng, lambda: eng.kv_park(0))                      # empty
        refused_quietly(eng, lambda: eng.kv_park(2 * B))                  # bad seq
        refused_quietly(eng, lambda: eng.kv_unpark(h, 1))                 # target not empty
        refused_quietly(eng, lambda: eng.kv_unpark(h, -1))
        refused_quietly(eng, lambda: eng.kv_unpark(h + 100, 2))           # no such record
        refused_quietly(eng, lambda: eng.kv_park_release(h + 100))
        eng.kv_unpark(h, 4)                                               # another index, a negative-stream one
        assert eng.kv_len(4) == 200 and eng.kv_pages_free() == free0 and same_kv(kv_all(eng, 4, 0, 200), src)
        msg = eng.lib.vv_last_error()
        assert eng.kv_parked_pages(h) == -1 and eng.lib.vv_last_error() == msg      # used up; a query records no error
        refused_quietly(eng, lambda: eng.kv_unpark(h, 2))
        # the next decode append lands where it would have without parking: sequence 0 prefilled again is the reference
        eng.lm_prefill(0, e)
        eng.kv_set_len(0, 200)
        x = torch.randn(dc.hidden_size, generator=torch.Generator().manual_seed(3)).cuda()
        modes = [1, 0, 0, 0, 1, 0]
        eng.set_row_mode(modes)
        with torch.cuda.stream(eng.stream):
            eng.embeds.zero_()
            eng.embeds[0].copy_(x)
            eng.embeds[4].copy_(x)
        eng.lm_decode()
        eng.kv_commit(modes)
        eng.set_row_mode([1] * (2 * B))
        eng.sync()
        assert eng.kv_len(0) == eng.kv_len(4) == 201
        assert same_kv(kv_all(eng, 0, 0, 201), kv_all(eng, 4, 0, 201))
        # release gives the pages back; kv_init drops every record
        h2 = eng.kv_park(4)
        eng.kv_park_release(h2)
        assert eng.kv_parked_pages(h2) == -1
        refused_quietly(eng, lambda: eng.kv_park_release(h2))
        h3 = eng.kv_park(0)
        for s in range(2 * B):
            eng.kv_set_len(s, 0)
        assert eng.kv_pages_free() == total - 4
        eng.kv_init(4096)
        assert eng.kv_parked_pages(h3) == -1 and eng.kv_pages_free() == eng.kv_pages
        refused_quietly(eng, lambda: eng.kv_unpark(h3, 0))
    finally:
        eng.close()


def test_park_keeps_shared_prefix_and_its_immutability():
    m, cfg, tok = make_model("tiny", 3, parts=PARTS, prefill_impl="native")
    eng = m.engine
    try:
        dc = cfg.decoder_config
        eng.kv_init(4096)
        e = embeds(cfg, 230, 4)
        eng.lm_prefill(0, e[:192])
        eng.kv_set_len(0, 192)
        hp = eng.kv_prefix_create(0, 192)
        eng.kv_prefix_attach(hp, 1)
        eng.lm_prefill(1, e[192:], pos0=192)
        eng.kv_set_len(1, 230)
        src = kv_all(eng, 1, 0, 230)
        free0 = eng.kv_pages_free()
        h = eng.kv_park(1)
        eng.kv_prefix_release(hp)                                         # the parked record still holds the shared pages
        eng.kv_set_len(0, 0)
        assert eng.kv_parked_pages(h) == 4
        eng.kv_unpark(h, 5)
        assert eng.kv_len(5) == 230 and eng.kv_seq_pages(5) == 4 and same_kv(kv_all(eng, 5, 0, 230), src)
        kz = torch.zeros(4, dc.num_key_value_heads, dc.head_dim, dtype=torch.bfloat16, device=eng.device)
        refused_quietly(eng, lambda: eng.lm_prefill(5, embeds(cfg, 10, 2), pos0=100))
        refused_quietly(eng, lambda: eng.kv_write(5, 0, 190, kz, kz))
        refused_quietly(eng, lambda: eng.kv_delete(5, 5))
        refused_quietly(eng, lambda: eng.kv_set_len(5, 100))
        eng.sync()
        assert same_kv(kv_all(eng, 5, 0, 230), src)
        eng.kv_set_len(5, 0)
        assert eng.kv_pages_free() == eng.kv_pages and free0 < eng.kv_pages
    finally:
        eng.close()


@pytest.mark.parametrize("preset", ["tiny", "1.5b-l2"])
def test_codec_state_save_load(preset):
    m, cfg, tok = make_model(preset, 3, parts=PARTS, prefill_impl="native")
    eng = m.engine
    try:
        g = torch.Generator().manual_seed(1)
        eng.codec_state_reset()
        for _ in range(3):                                               # rows 0 and 2 build up history from different latents
            with torch.cuda.stream(eng.stream):
                eng.latent.copy_(torch.randn(eng.B, 64, generator=g).cuda())
            eng.upload_frame_inputs(torch.zeros(2, 64), [0, 2])
            eng.codec_decode()
            eng.semantic_encode()
        n = eng.lib.vv_codec_state_floats(eng.h)
        save = lambda r: (eng.codec_state_save(r), eng.sync())[0]      # valid once the engine stream has run the copy
        a = save(0)
        assert a.numel() == n > 0 and a.abs().sum() > 0
        eng.codec_state_zero([0])
        eng.codec_state_load(0, a)
        assert torch.equal(save(0), a)                                   # round trip
        eng.codec_state_load(1, a)                                       # row 0's state on row 1
        assert torch.equal(save(1), a)
        assert not torch.equal(save(2), a)
        refused_quietly(eng, lambda: eng.codec_state_load(eng.B, a))
        refused_quietly(eng, lambda: eng.codec_state_save(-1))
        with torch.cuda.stream(eng.stream):                              # one more frame, the same latent on rows 0 and 1
            lat = torch.randn(64, generator=g).cuda()
            eng.latent[0].copy_(lat)
            eng.latent[1].copy_(lat)
        eng.upload_frame_inputs(torch.zeros(2, 64), [0, 1])
        eng.codec_decode()
        eng.semantic_encode()
        eng.sync()
        # the moved row continues as the row it came from (the T >= 40 codec GEMMs add split-K partials with fp32 atomics, so two rows
        # agree to rounding, not bit for bit)
        for x in (eng.audio, eng.feat):
            d = float((x[0] - x[1]).abs().max()) / float(x[0].abs().max())
            assert d < 1e-5, d
    finally:
        eng.close()


# ---- queue ------------------------------------------------------------------------------------------------------------------------------
def serve_with_priorities(m, low, high):
    """Serve `low` (priority 0); after the first frame submit `high` (priority 1), which parks the rows it finds no free row for.
    Returns the outputs in submission order, the queue and the parked requests."""
    from vibevoice_b200.serving import RequestQueue
    eng = m.engine
    q = RequestQueue(m, max_total_tokens=32768)
    sub = lambda r, p: q.submit(r["inputs"], cfg_scale=r["cfg_scale"], steps=r["steps"], solver=r["solver"], max_new_tokens=r["max_new_tokens"],
                                seed=r["seed"], voice_preset=r.get("preset"), priority=p)
    rids = [sub(r, 0) for r in low]
    frame, park, parked = q._frame, q._park, []

    def counted():
        done = frame()
        if len(rids) == len(low):
            rids.extend(sub(r, 1) for r in high)
        return done

    def logged(r):
        parked.append(q._rows[r].req)
        park(r)
    q._frame, q._park = counted, logged
    got = dict(q.run())
    assert sorted(got) == sorted(rids) and q._pages_used == 0
    assert q.parks >= 1, "no row was parked"
    for s in range(2 * eng.B):
        eng.kv_set_len(s, 0)
    return [got[i] for i in rids], q, parked


@pytest.mark.parametrize("preset,B", [("tiny", 2), ("tiny", 8), ("1.5b-l2", 2), ("1.5b-l2", 8)])
def test_queue_with_priorities_matches_solo(preset, B):
    m, cfg, tok = make_model(preset, B, prefill_impl="native")
    eng = m.engine
    try:
        pre = prefix_inputs(cfg, tok, 11, 2, 90)
        P = m.voice_preset(pre, seed=21)
        low = plain_requests(cfg, tok, B, B, seed=B, voices=False)
        for i, r in enumerate(low):                                      # long scripts; every other one on the preset
            r["max_new_tokens"] = 24 + 3 * i
            if i % 2 == 0:
                r["inputs"], r["preset"] = full_request(pre, cfg, tok, 6 + i, 80 + i), P
            else:
                r["preset"] = None
        high = plain_requests(cfg, tok, B, B, seed=100 + B, voices=False)
        for i, r in enumerate(high):
            r["max_new_tokens"], r["preset"] = 4 + i % 3, None
        got, q, parked = serve_with_priorities(m, low, high)
        assert any(req.preset is not None for req in parked), [req.rid for req in parked]
        P.release()
        assert eng.kv_pages_free() == eng.kv_pages
        for i, (r, out) in enumerate(zip(low + high, got)):
            assert_same(out, solo_preset(m, tok, r), (preset, B, i))
    finally:
        eng.close()
