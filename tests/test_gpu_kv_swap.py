"""`-m gpu` tests of swapped parked records (`vv_kv_swap_*`): the host image's layout bit for bit, pages freed and reused while a
record is on the host, a bit-identical swap-in on another sequence index, shared prefix pages that stay in the pool, launches of more
than 32 pages, refusals, and `RequestQueue(host_swap_bytes=...)` on a pool sized for its live rows against solo `generate()`."""

import pytest
import torch

from test_gpu_preempt import refused_quietly
from test_gpu_queue import requests as plain_requests
from test_gpu_voice_preset import PARTS, assert_same, embeds, full_request, kv_all, make_model, prefix_inputs, same_kv, solo_preset

from vibevoice_b200 import _native as NV

pytestmark = pytest.mark.gpu


def host_image(eng, buf, n_pages):
    """the swap buffer as [page, layer, K/V, kv_heads, 64, head_dim] bf16"""
    dc = eng.config.decoder_config
    return buf.view(torch.bfloat16).view(n_pages, dc.num_hidden_layers, 2, dc.num_key_value_heads, 64, dc.head_dim)


def assert_image(eng, img, src, first_page, n_tokens):
    """positions [64 * first_page, n_tokens) of `src` (kv_all from position 0) equal the host image, page by page"""
    for l, (k, v) in enumerate(src):
        for t0 in range(64 * first_page, n_tokens, 64):
            t1 = min(t0 + 64, n_tokens)
            p = t0 // 64 - first_page
            for kv, x in enumerate((k, v)):
                assert torch.equal(img[p, l, kv, :, :t1 - t0].cpu(), x[t0:t1].transpose(0, 1).cpu()), (l, p, kv)


def refused_with(eng, fn, code):
    """refused with return code `code`, an error message and no launch"""
    n = eng.launch_count()
    with pytest.raises(NV.VVError, match=r"failed \(%d\)" % code):
        fn()
    assert eng.launch_count() == n and eng.lib.vv_last_error()


def test_swap_runtime():
    m, cfg, tok = make_model("tiny", 3, parts=PARTS, prefill_impl="native")
    eng = m.engine
    try:
        B, dc = eng.B, cfg.decoder_config
        eng.kv_init(1024)
        e = embeds(cfg, 200, 1)
        eng.lm_prefill(0, e)
        eng.kv_set_len(0, 200)
        src = kv_all(eng, 0, 0, 200)
        h = eng.kv_park(0)
        free0 = eng.kv_pages_free()
        buf = eng.kv_swap_out(h)
        eng.sync()
        assert eng.kv_pages_free() == free0 + 4 and eng.kv_parked_pages(h) == 0
        assert eng.kv_swap_bytes(h) == 4 * eng.kv_page_bytes == buf.numel()
        assert_image(eng, host_image(eng, buf, 4), src, 0, 200)
        # refusals: nothing launched, the free count unchanged, an error recorded
        pageable = torch.empty(buf.numel(), dtype=torch.uint8)
        n = buf.numel()
        for fn, code in ((lambda: eng.kv_swap_out(h), -3),                                     # already swapped
                         (lambda: eng.kv_unpark(h, 1), -3),                                    # swapped
                         (lambda: eng.kv_swap_in(h, pageable), -1),                            # not page-locked
                         (lambda: eng.kv_swap_in(h, buf[:n - 16]), -1),                        # too small
                         (lambda: eng.kv_swap_in(h + 100, buf), -1),                           # dead handle
                         (lambda: NV.check(eng.lib.vv_kv_swap_in(eng.h, h, None, n, eng.s), "vv_kv_swap_in"), -1)):   # null
            refused_with(eng, fn, code)
            assert eng.kv_pages_free() == free0 + 4
        msg = eng.lib.vv_last_error()
        assert eng.kv_swap_bytes(h + 100) == -1 and eng.lib.vv_last_error() == msg           # a query records no error
        # the freed pages go to another sequence and are overwritten there
        eng.lm_prefill(1, embeds(cfg, 300, 2))
        eng.kv_set_len(1, 300)
        other = kv_all(eng, 1, 0, 300)
        # not enough free pages: VV_ERR_NOMEM, nothing changes; once pages are free the same swap-in succeeds
        fill = 64 * (eng.kv_pages_free() - 2)
        eng.lm_prefill(2, embeds(cfg, fill, 3))
        eng.kv_set_len(2, fill)
        full = eng.kv_pages_free()
        assert full < 4
        refused_with(eng, lambda: eng.kv_swap_in(h, buf), -4)
        assert "needs 4 pages" in eng.lib.vv_last_error().decode() and eng.kv_pages_free() == full
        eng.kv_set_len(2, 0)
        eng.kv_swap_in(h, buf)
        assert eng.kv_parked_pages(h) == 4 and eng.kv_swap_bytes(h) == 4 * eng.kv_page_bytes
        refused_with(eng, lambda: eng.kv_swap_in(h, buf), -3)                                   # resident
        eng.kv_unpark(h, 4)                                                                     # another index
        assert eng.kv_len(4) == 200 and same_kv(kv_all(eng, 4, 0, 200), src)
        assert same_kv(kv_all(eng, 1, 0, 300), other)
        # the next decode append matches a sequence that was never swapped: sequence 0 prefilled again
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
        # release of a swapped record, and vv_kv_init drops swapped records
        h2 = eng.kv_park(4)
        eng.kv_swap_out(h2)
        eng.kv_park_release(h2)
        assert eng.kv_swap_bytes(h2) == -1
        h3 = eng.kv_park(0)
        b3 = eng.kv_swap_out(h3)
        for s in range(2 * B):
            eng.kv_set_len(s, 0)
        assert eng.kv_pages_free() == eng.kv_pages
        eng.kv_init(1024)
        assert eng.kv_swap_bytes(h3) == -1
        refused_quietly(eng, lambda: eng.kv_swap_in(h3, b3))
    finally:
        eng.close()


def test_swap_keeps_shared_prefix():
    m, cfg, tok = make_model("tiny", 3, parts=PARTS, prefill_impl="native")
    eng = m.engine
    try:
        eng.kv_init(4096)
        e = embeds(cfg, 230, 4)
        eng.lm_prefill(0, e[:192])
        eng.kv_set_len(0, 192)
        hp = eng.kv_prefix_create(0, 192)
        eng.kv_prefix_attach(hp, 1)
        eng.lm_prefill(1, e[192:], pos0=192)
        eng.kv_set_len(1, 230)
        src = kv_all(eng, 1, 0, 230)
        h = eng.kv_park(1)
        free0 = eng.kv_pages_free()
        buf = eng.kv_swap_out(h)                                          # only page 3 (positions 192..229) moves
        eng.sync()
        assert buf.numel() == eng.kv_page_bytes and eng.kv_pages_free() == free0 + 1 and eng.kv_parked_pages(h) == 3
        assert_image(eng, host_image(eng, buf, 1), src, 3, 230)
        eng.kv_prefix_release(hp)
        eng.kv_set_len(0, 0)
        assert eng.kv_pages_free() == free0 + 1                           # the swapped record still holds the 3 shared pages
        eng.lm_prefill(2, embeds(cfg, 400, 5))                            # reuses the freed pages
        eng.kv_set_len(2, 400)
        eng.kv_swap_in(h, buf)
        eng.kv_unpark(h, 5)
        assert eng.kv_len(5) == 230 and eng.kv_seq_pages(5) == 4 and same_kv(kv_all(eng, 5, 0, 230), src)
        refused_quietly(eng, lambda: eng.kv_set_len(5, 100))             # the shared positions stay immutable
        for s in (2, 5):
            eng.kv_set_len(s, 0)
        assert eng.kv_pages_free() == eng.kv_pages
    finally:
        eng.close()


def test_swap_more_than_32_pages():
    """34 private pages at the 1.5B layer shapes: two launches, the second one starting at private page 32."""
    m, cfg, tok = make_model("1.5b-l2", 2, parts=PARTS, prefill_impl="native")
    eng = m.engine
    try:
        eng.kv_init(8192)
        L = 33 * 64 + 10
        eng.lm_prefill(0, embeds(cfg, L, 6))
        eng.kv_set_len(0, L)
        src = kv_all(eng, 0, 0, L)
        h = eng.kv_park(0)
        n0 = eng.launch_count()
        buf = eng.kv_swap_out(h)
        assert eng.launch_count() == n0 + 2 and buf.numel() == 34 * eng.kv_page_bytes
        eng.sync()
        assert_image(eng, host_image(eng, buf, 34), src, 0, L)
        eng.lm_prefill(1, embeds(cfg, L, 7))                              # overwrite the freed pages
        eng.kv_set_len(1, L)
        eng.kv_swap_in(h, buf)
        eng.kv_unpark(h, 3)
        assert same_kv(kv_all(eng, 3, 0, L), src)
    finally:
        eng.close()


# ---- queue ------------------------------------------------------------------------------------------------------------------------------
def pages_of(r, shared):
    L0 = r["inputs"]["input_ids"].shape[1]
    ms = min(r["max_new_tokens"], 2 * L0)
    return (L0 + ms + 2 + 63) // 64 + (ms + 2 + 63) // 64 - shared


@pytest.mark.parametrize("preset,B", [("tiny", 2), ("tiny", 8), ("1.5b-l2", 2), ("1.5b-l2", 8)])
def test_queue_with_swap_matches_solo(preset, B):
    """B low-priority rows fill a pool sized for them alone; B high-priority requests arrive after the first frame and can only be
    admitted by swapping rows out.  Every request equals its solo run, and the pool is whole once the queue drains."""
    from vibevoice_b200.serving import RequestQueue
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
        live = sum(pages_of(r, P.pages if r["preset"] is not None else 0) for r in low) + P.pages
        q = RequestQueue(m, max_total_tokens=64 * (live - 2 * B), host_swap_bytes=1 << 34)
        assert q._budget == live
        sub = lambda r, p: q.submit(r["inputs"], cfg_scale=r["cfg_scale"], steps=r["steps"], solver=r["solver"],
                                    max_new_tokens=r["max_new_tokens"], seed=r["seed"], voice_preset=r.get("preset"), priority=p)
        rids = [sub(r, 0) for r in low]
        frame, swap_out, swapped = q._frame, q._swap_out, []

        def counted():
            done = frame()
            if len(rids) == len(low):
                rids.extend(sub(r, 1) for r in high)
            return done
        q._frame = counted
        q._swap_out = lambda row: (swapped.append(row.req), swap_out(row))
        got = dict(q.run())
        assert sorted(got) == sorted(rids) and q._pages_used == 0 and q.host_bytes_used == 0
        assert q.swaps > 0 and any(req.preset is not None for req in swapped), [req.rid for req in swapped]
        for s in range(2 * B):
            eng.kv_set_len(s, 0)
        P.release()
        assert eng.kv_pages_free() == eng.kv_pages
        for i, (r, rid) in enumerate(zip(low + high, rids)):
            assert_same(got[rid], solo_preset(m, tok, r), (preset, B, i))
    finally:
        eng.close()
