"""CPU tests of `RequestQueue(host_swap_bytes=...)` on the engine stand-in, extended here with swapped parked records: that a zero or
unused host budget changes no engine call, that with a pool sized for the live rows a higher-priority request is admitted at the next
frame boundary only when swapping is on, which requests are swapped, that swapped requests resume with their solo results, and that
the pool and host charges stay exact after every frame, through `cancel` and an early exit from `run()`."""
import copy
import random

import pytest
import torch

from test_preempt_host import ParkFakeEngine, assert_same, request, solo

PAGE_BYTES = 1000


class SwapFakeEngine(ParkFakeEngine):
    """The parking stand-in plus the swap ABI: a swapped record's K/V cache object moves into a host-side copy and comes back on
    swap-in.  It counts pool pages the way the runtime does (a sequence holds ceil(entries / 64) pages, the first shared / 64 of them
    a prefix's) and refuses a swap-in the pool cannot hold.  Every call, with its scalar arguments, is recorded in `abi_calls`."""

    kv_page_bytes = PAGE_BYTES

    def kv_init(self, total_tokens):
        super().kv_init(total_tokens)
        self.shared = [0] * (2 * self.B)
        self.park_shared, self.host = {}, {}

    def __getattribute__(self, name):
        v = object.__getattribute__(self, name)
        if name.startswith("_") or not callable(v) or name in ("pool_used", "kv_len", "kv_seq_pages"):
            return v
        calls = object.__getattribute__(self, "__dict__").setdefault("abi_calls", [])

        def logged(*a, **k):
            calls.append((name,) + tuple(x for x in a if isinstance(x, (int, float, str))))
            return v(*a, **k)
        return logged

    # page accounting
    def kv_seq_pages(self, seq):
        return (len(self.kv[seq]) + 63) // 64

    def _private(self, h):
        if h in self.host:
            return (len(self.host[h]) + 63) // 64 - self.park_shared[h] // 64
        return (len(self.parked[h]) + 63) // 64 - self.park_shared[h] // 64

    def pool_used(self):
        seqs = sum(self.kv_seq_pages(s) - self.shared[s] // 64 for s in range(2 * self.B))
        return seqs + sum(self._private(h) for h in self.parked) + sum(self.prefix_pages.values())

    def kv_set_len(self, seq, n):
        super().kv_set_len(seq, n)
        if n == 0:
            self.shared[seq] = 0

    def kv_prefix_create(self, seq, n):
        self.shared[seq] = max(self.shared[seq], n)
        return super().kv_prefix_create(seq, n)

    def kv_prefix_attach(self, h, seq):
        super().kv_prefix_attach(h, seq)
        self.shared[seq] = self.prefixes[h][0]

    def kv_park(self, seq):
        h = super().kv_park(seq)
        self.park_shared[h], self.shared[seq] = self.shared[seq], 0
        return h

    def kv_unpark(self, h, seq):
        assert h not in self.host, "unpark of a swapped record"
        super().kv_unpark(h, seq)
        self.shared[seq] = self.park_shared.pop(h)

    def kv_park_release(self, h):
        if h in self.host:
            del self.host[h]
            self.log.append(("park_release", h))
        else:
            super().kv_park_release(h)
        del self.park_shared[h]

    # swap
    def kv_swap_bytes(self, h):
        return self._private(h) * PAGE_BYTES if h in self.park_shared else -1

    def kv_swap_out(self, h):
        assert h in self.parked, "swap-out of a swapped or dead record"
        self.host[h] = copy.deepcopy(self.parked.pop(h))
        self.log.append(("swap_out", h))
        return self.host[h]

    def kv_swap_in(self, h, buf):
        assert h in self.host and buf is self.host[h]
        assert self.pool_used() + self._private(h) <= self.kv_pages, "swap-in beyond the pool"
        self.parked[h] = self.host.pop(h)
        self.log.append(("swap_in", h))


@pytest.fixture(scope="module")
def setup():
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference, VoicePreset
    from vibevoice_b200.synth import SynthTokenizer, synth_state_dict
    cfg = preset_config("tiny")
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, 1234, torch.float32)

    def make(B):
        m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=B, prefill_impl="native")
        m.engine = SwapFakeEngine(cfg, m._valid_ids(tok), B, weights=sd)
        m.engine.log = []
        m._scale, m._bias = float(sd["model.speech_scaling_factor"]), float(sd["model.speech_bias_factor"])
        return m

    def preset(m, Lp, seed):
        ids = torch.randint(0, cfg.decoder_config.vocab_size - 20, (Lp,), generator=torch.Generator().manual_seed(seed))
        return VoicePreset(m, ids, m.engine.embed_gather(ids).clone(), (None, None))
    return cfg, tok, make, preset


def check_charges(q):
    """the pool charge is the live and resident-parked requests' worst case, the host charge the swapped requests' bytes, and the
    pages the pool really holds stay within the charge"""
    live = [row.req for row in q._rows if row is not None]
    resident = [w for w in q._waiting if w.parked is not None and w.parked.host is None]
    swapped = [w for w in q._waiting if w.parked is not None and w.parked.host is not None]
    assert q._pages_used == sum(r.pages for r in live + resident), (q._pages_used, [r.rid for r in live + resident])
    assert q.host_bytes_used == sum(w.parked.host_bytes for w in swapped) <= max(q._host_budget, 0)
    eng = q.eng
    assert eng.pool_used() <= q._pages_used + q.preset_pages() + 2 * q.B, (eng.pool_used(), q._pages_used, q.preset_pages())
    assert q._pages_used + q.preset_pages() <= q._budget


def drive(q, first, arrivals=None, after_frame=None):
    """test_preempt_host.drive with the charges checked after every frame and the live request ids recorded per frame: returns
    ({rid: output}, [rids in submit order], [rids holding a row when frame n starts, n = 1, 2, ...])"""
    rids = [q.submit(**r) for r in first]
    frame, live = q._frame, []

    def counted():
        live.append([row.req.rid for row in q._rows if row is not None])
        done = frame()
        n = len(live)
        for r in (arrivals or {}).get(n, []):
            rids.append(q.submit(**r))
        if after_frame is not None:
            done += after_frame(n, [rid for rid, _ in done])
        check_charges(q)
        return done
    q._frame = counted
    got = dict(q.run())
    return got, rids, live


def swapped_rows(m):
    """positive sequence indices whose records were swapped out, in order"""
    seq_of, out = {}, []
    park_no = 0
    for e in m.engine.log:
        if e[0] == "park":
            park_no += 1
            seq_of[park_no] = e[1]
        elif e[0] == "swap_out" and seq_of[e[1]] < m.engine.B:
            out.append(seq_of[e[1]])
    return out


@pytest.mark.parametrize("case", ["newest_of_equal", "lowest_first", "resume_other_row", "mixed"])
def test_zero_or_unused_host_budget_changes_nothing(setup, case):
    """The priority scenarios of test_preempt_host.py: the same engine calls with host_swap_bytes omitted, 0, or large on a pool that
    never runs short."""
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, preset = setup
    long = lambda s, p, L=6: request(cfg, tok, L, 40, s, priority=p)
    if case == "newest_of_equal":
        first, arrive = [long(1, 0), long(2, 0)], {3: [long(9, 1)]}
    elif case == "lowest_first":
        first, arrive = [long(1, 0)], {1: [long(2, 1)], 3: [long(9, 2)]}
    elif case == "resume_other_row":
        first, arrive = [request(cfg, tok, 6, 8, 1, priority=0), request(cfg, tok, 8, 30, 2, priority=0)], {2: [long(3, 1, 7)]}
    else:
        rnd = random.Random(4)
        first = [long(10 + i, 0, rnd.randint(4, 14)) for i in range(3)]
        arrive = {f: [long(20 + f, rnd.choice([0, 1, 2]), rnd.randint(4, 14))] for f in sorted(rnd.sample(range(2, 14), 4))}
    runs = []
    for kw in ({}, {"host_swap_bytes": 0}, {"host_swap_bytes": 1 << 40}):
        m = make(2)
        q = RequestQueue(m, max_total_tokens=4096, **kw)
        got, rids, _ = drive(q, first, arrive)
        assert q.swaps == 0 and q.parks >= 1
        runs.append((m.engine.abi_calls, [got[r].sequences.tolist() for r in rids]))
    assert runs[0] == runs[1] == runs[2]


def live_only(cfg, tok, hi_seed=9):
    """two 40-step rows (3 pages each) on a pool whose request budget is 6 pages (max_total_tokens=128): a third request (2 pages)
    does not fit beside them"""
    low = [request(cfg, tok, 24, 40, s, priority=0) for s in (1, 2)]
    hi = request(cfg, tok, 10, 8, hi_seed, priority=1)
    return low, hi


@pytest.mark.parametrize("swap", [False, True])
def test_live_rows_pool(setup, swap):
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, _ = setup
    m, solo_m = make(2), make(2)
    q = RequestQueue(m, max_total_tokens=128, host_swap_bytes=10 * PAGE_BYTES if swap else 0)
    assert q._budget == 6
    low, hi = live_only(cfg, tok)
    got, rids, live = drive(q, low, {3: [hi]})
    admitted = next(n for n, rows in enumerate(live, 1) if rids[2] in rows)
    first_done = next(n for n, rows in enumerate(live, 1) if not set(rids[:2]) <= set(rows))
    if swap:
        assert admitted == 4 and q.swaps == 1 and q.parks == 1                # the next frame boundary after its arrival
        assert swapped_rows(m) == [1]                                       # the newer of the two backlog rows
        kinds = [e[0] for e in m.engine.log if e[0] in ("park", "swap_out", "swap_in", "unpark")]
        assert kinds.index("swap_in") > max(i for i, k in enumerate(kinds) if k == "swap_out") and kinds[-1] == "unpark"
    else:
        assert admitted == first_done > 4 and q.swaps == 0 and q.parks == 0  # it waits until a backlog row has finished
    assert sorted(got) == sorted(rids) and q._pages_used == 0 and q.host_bytes_used == 0
    assert not m.engine.parked and not m.engine.host
    for rid, r in zip(rids, low + [hi]):
        assert_same(got[rid], solo(solo_m, tok, r), rid)


@pytest.mark.parametrize("host,want", [(7000, [2]), (3000, [1]), (1500, [0]), (500, [])])
def test_swap_candidates(setup, host, want):
    """The priority-1 request takes row 0, then the priority-0 ones rows 1 and 2 (row 2, admitted last, is the victim).  A priority-2
    head of 4 pages arrives and fits once any one request is swapped.  Row 2 holds 4000 host bytes, row 1 2000 and row 0 1000.  The
    victim goes first when the host has room for it; else the running rows follow, lower priority first (row 1, then row 0), each
    skipped when the host has no room for it; with room for none nothing is swapped and the head waits."""
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, _ = setup
    m = make(3)
    q = RequestQueue(m, max_total_tokens=6 * 64, host_swap_bytes=host)
    first = [request(cfg, tok, 20, 40, 1, priority=0), request(cfg, tok, 200, 40, 2, priority=0), request(cfg, tok, 20, 40, 3, priority=1)]
    hi = request(cfg, tok, 80, 50, 4, priority=2)
    seen = {}

    def look(n, done):
        if n == 3:
            seen["bytes"] = [q._private_bytes(q._rows[r]) for r in range(3)]
        return []
    got, rids, live = drive(q, first, {3: [hi]}, after_frame=look)
    assert seen["bytes"] == [1000, 2000, 4000]
    assert swapped_rows(m) == want and q.swaps == len(want), m.engine.log
    admitted = next(n for n, rows in enumerate(live, 1) if rids[3] in rows)
    if want:
        assert admitted == 4 and q.parks == 1
    else:
        assert admitted > 4 and q.parks == 0
    assert sorted(got) == sorted(rids) and not m.engine.parked and not m.engine.host


@pytest.mark.parametrize("seed", [0, 1])
def test_swapped_requests_match_solo(setup, seed):
    """Random scripts, priorities and arrivals over 2 rows on a pool sized for the live rows, some requests on a voice preset (whose
    shared page stays charged once while its holders are swapped): every request equals its solo run."""
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, preset = setup
    rnd = random.Random(seed)
    m, solo_m = make(2), make(2)
    P = preset(m, 70, 5)
    solo_presets = {P: preset(solo_m, 70, 5)}
    q = RequestQueue(m, max_total_tokens=3 * 64, host_swap_bytes=100 * PAGE_BYTES)
    mk = lambda i, pr: request(cfg, tok, rnd.randint(12, 24), rnd.randint(20, 40), 100 * seed + i, priority=pr,
                               preset=P if i % 2 == 0 else None, steps=rnd.choice([1, 2]), cfg_scale=rnd.choice([1.0, 1.3]))
    first = [mk(i, 0) for i in range(3)]
    arrivals, i = {}, 3
    for f in sorted(rnd.sample(range(2, 14), 4)):
        arrivals[f] = [mk(i, rnd.choice([1, 2, 2]))]
        i += 1
    reqs = first + [r for f in sorted(arrivals) for r in arrivals[f]]
    swap_out, swapped = q._swap_out, []
    q._swap_out = lambda row: (swapped.append(row.req), swap_out(row))
    got, rids, _ = drive(q, first, arrivals)
    assert sorted(got) == sorted(rids) and q._pages_used == 0 and q.host_bytes_used == 0
    assert any(r.preset is not None for r in swapped), [r.rid for r in swapped]
    assert q.swaps >= 1 and not m.engine.parked and not m.engine.host
    assert len(events(m, "swap_in")) == len(events(m, "swap_out"))
    for rid, r in zip(rids, reqs):
        assert_same(got[rid], solo(solo_m, tok, r, solo_presets), (seed, rid))


def events(m, kind):
    return [e[1] for e in m.engine.log if e[0] == kind]


def test_cancel_a_swapped_request_and_leave_early(setup):
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, _ = setup
    m, solo_m = make(2), make(2)
    q = RequestQueue(m, max_total_tokens=128, host_swap_bytes=10 * PAGE_BYTES)
    low, hi = live_only(cfg, tok)
    out = {}

    def act(n, done):
        if n == 4:                                       # rid 1 was parked and swapped for rid 2 at the boundary after frame 3
            sw = [w.rid for w in q._waiting if w.parked is not None and w.parked.host is not None]
            assert sw == [1] and q.host_bytes_used > 0
            out["swapped"] = q.cancel(1)
            assert q.host_bytes_used == 0
        return []
    got, rids, _ = drive(q, low, {3: [hi]}, after_frame=act)
    assert sorted(got) == [0, 2] and not m.engine.parked and not m.engine.host and q._pages_used == 0
    assert len(events(m, "park_release")) >= 1 and not events(m, "swap_in")
    o, want = out["swapped"], solo(solo_m, tok, low[1])
    n = o.sequences.shape[1]
    assert torch.equal(o.sequences, want.sequences[:, :n])

    # leaving run() early, with a swapped request waiting, releases its records and host copies
    m = make(2)
    q = RequestQueue(m, max_total_tokens=128, host_swap_bytes=10 * PAGE_BYTES)
    for r in low:
        q.submit(**r)
    frame, frames = q._frame, [0]

    def counted():
        frames[0] += 1
        if frames[0] == 4:
            q.submit(**hi)
        return frame()
    q._frame = counted
    it = q.run()
    for _ in it:
        break
    it.close()
    assert q.swaps == 1 and q.host_bytes_used == 0 and q._pages_used == 0
    assert not m.engine.parked and not m.engine.host and not m.engine.park_shared
