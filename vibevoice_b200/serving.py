"""A queue of requests served on one GPU's B rows: a row that finishes takes the next waiting request mid-generation.

A static `generate()` batch runs until its longest row ends, and the frame cost is dominated by the weight stream, not by the number of
live rows, so in a static batch the useful share of the work is mean length / max length.  `RequestQueue` keeps the rows busy instead:

    q = RequestQueue(model, max_total_tokens=...)
    rid = q.submit(inputs, cfg_scale=1.3, steps=10, solver="dpmsolver++", max_new_tokens=None, max_length_times=2, seed=1234)
    for rid, out in q.run():          # VibeVoiceGenerationOutput per request, in completion order
        ...

Each frame runs the per-row loop body of `modeling.generate` (refresh_negative=True) for every live row, each at its own step.  After the
frame the rows that finished are freed (both sequences to length 0, codec state zeroed) and waiting requests are admitted, highest
`priority` first and oldest first within a priority, while the KV pool can hold their worst case.  A waiting request that finds no free
row takes the row of a running request of strictly lower priority, which is parked between frames (its K/V pages, codec state and next
input set aside, `RequestQueue` docstring) and resumes later where it stopped.  Sampler settings are per row (`Engine.set_row_sampler`):
every row pays the largest step count of the requests in the queue per frame.

Results do not depend on batch-mates or on being parked: a request's output equals `torch.manual_seed(seed); model.generate(<that
request alone>, ...)` with `set_ddpm_inference_steps(steps)` and that solver.  Each request has its own CPU generator (diffusion noise, `randn(2, 64)[:1]` per
diffusion frame) and device generator (voice-prompt noise, then SDE step noise), drawn in the solo run's order.

`StreamingRequestQueue` does the same for the streaming-0.5B variant (`streaming.py`), with per-request audio streamers and text that
arrives while the request speaks (`push_text`).
"""
from __future__ import annotations

import bisect
import collections
from dataclasses import dataclass, field
from typing import Any, Deque, Iterator, List, Optional, Tuple

import torch

from . import _native as N
from .modeling import ForcedTokenScript, VibeVoiceGenerationOutput

SOLVERS = ("dpmsolver++", "sde-dpmsolver++")


@dataclass
class _Request:
    rid: int
    ids: torch.Tensor                   # [L0] prompt as given (left padding included)
    keep: torch.Tensor                  # [L0] bool attention mask
    voice: Optional[Tuple[Any, Any, torch.Tensor]]    # (speech_tensors, speech_masks, speech_input_mask [L0]) or None
    cfg_scale: float
    steps: int
    solver: str
    seed: int
    max_length: int
    max_steps: int
    max_step_per_sample: int
    pages: int                          # worst-case KV pages of both sequences (with a preset: those outside its shared pages)
    preset: Any = None                  # VoicePreset or None
    priority: int = 0
    parked: Optional["_Row"] = None     # the row state of a request parked mid-generation (its pages stay charged)

    def key(self):
        """waiting order: highest priority first, then submission order"""
        return (-self.priority, self.rid)


@dataclass
class _Row:
    req: _Request
    gen_cpu: torch.Generator
    gen_dev: torch.Generator
    order: int                          # admission order (prefill progress goes oldest first)
    embeds: Optional[torch.Tensor] = None   # prompt embeddings while the prefill runs
    done: int = 0                       # prompt tokens prefilled so far
    builds: bool = False                # prefilling its preset's shared pages, which become the preset's at `shared`
    prefix: Optional[int] = None        # handle of the shared pages the row holds (attached or built)
    hid: Optional[torch.Tensor] = None  # final-norm hidden state of the last prompt token
    step: int = -1                      # generation step of the next frame; -1 while admitting
    seq: List[int] = field(default_factory=list)
    finished: bool = False
    reach_max: bool = False
    audio: List[torch.Tensor] = field(default_factory=list)
    park: Optional[Tuple[int, Optional[int], torch.Tensor, torch.Tensor]] = None   # parked: (positive, negative KV handles, codec state,
                                                                                   # embeds rows r and B + r)
    host: Optional[List[Any]] = None    # swapped out: the pinned host copies of the parked records' private pages (positive, negative)
    host_bytes: int = 0                 # their size, charged against host_swap_bytes


class RequestQueue:
    """Continuous batching of single-script requests over the model's B rows (see the module docstring).

    `max_total_tokens` sizes the KV pool once, here (re-sizing it later would drop every sequence).  Prompts are prefilled on the model's
    prefill path: `TorchPrefill` when the model keeps one and does not default to the native prefill, else the native prefill
    (`vv_lm_prefill`) -- the token-by-token prefill of `generate()` cannot admit a row while other rows run.  A long prompt stalls every
    other row for its whole prefill; `max_prefill_tokens_per_frame` (native prefill only, rounded down to a multiple of 64) spreads it over
    frames, which is exact because the native prefill gives the same result for any chunking.

    Priorities: `submit(..., priority=p)` (default 0) serves waiting requests highest priority first, oldest first within a priority;
    with every priority equal the queue is first in, first out.  Between frames, when the request at the head finds no free row, a
    running request of strictly lower priority exists, and the head's worst case fits the pool beside everything already held, one row
    is preempted: the lowest-priority row, the most recently admitted among those, of the rows that have run at least one frame.  Its
    sequences' pages move into parked records (`Engine.kv_park`, no copy), its codec state and next-input embeddings are saved, and the
    request goes back to the waiting list at its own priority and submission order.  Parking alone frees no pages (they stay charged): a
    parked request needs only a free row to resume, on any row index, and a parked request whose pages keep the head waiting resumes
    ahead of it.  Being parked does not change a request's result.

    Swapping (`host_swap_bytes` > 0) makes preemption free pool pages too, so a pool sized for the live rows is enough.  When the head
    does not fit the pool between frames (a new request, or a swapped one that needs its pages back), the queue moves the private KV
    pages of lower-priority requests to pinned host memory (`Engine.kv_swap_out`) and uncharges their worst case.  Candidates, in order:
    the row the head preempts, if it has no free row; parked requests of strictly lower priority; then running rows of strictly lower
    priority that have run a frame (parked first); lowest priority first and most recently admitted first within a priority.  A candidate
    whose pages would overflow the host budget is skipped.  The queue swaps the shortest run of candidates after which the head fits, and
    nothing when none does.  A swapped request is charged its actual bytes against `host_swap_bytes`; it resumes once it is the head, a
    row is free and its worst case fits the pool again (`Engine.kv_swap_in`).  Shared preset pages, codec state and next-input embeddings
    stay on the device.  With `host_swap_bytes` = 0 nothing is swapped.

    `cancel(rid)` (between yields of `run()`) ends a waiting, admitting, running or parked request, frees its row and pages, and returns
    what it produced so far."""

    def __init__(self, model, max_total_tokens: int, max_prefill_tokens_per_frame: Optional[int] = None, host_swap_bytes: int = 0):
        eng = model.engine
        if eng is None or not eng.finalized:
            raise N.VVError("weights not loaded")
        self.model, self.eng, self.B = model, eng, eng.B
        self._native = model._prefill_impl == "native" or model._prefill is None
        self._chunk = None
        if max_prefill_tokens_per_frame is not None:
            if not self._native:
                raise ValueError("max_prefill_tokens_per_frame: the model prefills with TorchPrefill, which admits whole prompts; "
                                 "build it with prefill_impl=\"native\" to spread prompts over frames")
            if int(max_prefill_tokens_per_frame) < 64:
                raise ValueError("max_prefill_tokens_per_frame must be at least 64 (got %r)" % (max_prefill_tokens_per_frame,))
            self._chunk = int(max_prefill_tokens_per_frame) // 64 * 64
        eng.kv_init(int(max_total_tokens))
        self._budget = eng.kv_pages - 2 * self.B          # lm_decode keeps one page for every sequence's next entry
        self._waiting: List[_Request] = []                 # in _Request.key order
        self._next_rid = 0
        self._rows: List[Optional[_Row]] = [None] * self.B
        self._pages_used = 0                               # the live and parked rows' pages (shared prefixes: preset_pages())
        self._admitted = 0
        self._nmax = 0
        self._modes: Optional[List[int]] = None
        self.parks = 0                                     # rows preempted so far
        if int(host_swap_bytes) < 0:
            raise ValueError("host_swap_bytes must be >= 0 (got %r)" % (host_swap_bytes,))
        self._host_budget = int(host_swap_bytes)
        self.swaps = 0                                     # parked requests swapped out so far
        self.host_bytes_used = 0                           # host bytes of the swapped requests' pages

    # ---- requests ---------------------------------------------------------------------------------------------------------------------
    def submit(self, inputs, cfg_scale: float = 1.3, steps: int = 10, solver: str = "dpmsolver++", max_new_tokens: Optional[int] = None,
               max_length_times: float = 2, seed: int = 1234, generation_config=None, logits_processor=None, audio_streamer=None,
               stop_check_fn=None, refresh_negative: bool = True, voice_preset=None, priority: int = 0) -> int:
        """Queue one request; `inputs` is the processor output for ONE script (+ its voices).  Returns the request id `run()` reports.
        With `voice_preset` (`model.voice_preset`) the prompt must start with the preset's prefix: the request runs no voice encoding,
        attaches the preset's shared K/V pages (prefilling them first if they are not in the pool) and is prefilled natively from there;
        its result equals `generate(<that request>, voice_preset=voice_preset)`.  `priority`: a higher one is served first and may
        preempt running requests of lower priority (class docstring)."""
        if audio_streamer is not None:
            raise ValueError("audio_streamer is not supported by RequestQueue")
        if stop_check_fn is not None:
            raise ValueError("stop_check_fn is not supported by RequestQueue")
        if logits_processor is not None:
            procs = logits_processor if isinstance(logits_processor, (list, tuple)) else [logits_processor]
            if any(isinstance(p, ForcedTokenScript) for p in procs):
                raise ValueError("logits_processor: forced token scripts are not supported by RequestQueue")
            raise ValueError("logits_processor objects are not supported by RequestQueue")
        if not refresh_negative:
            raise ValueError("refresh_negative=False is not supported by RequestQueue")
        if generation_config is not None:
            g = dict(generation_config) if isinstance(generation_config, dict) else \
                {k: v for k, v in vars(generation_config).items() if not k.startswith("_")}
            if bool(g.get("do_sample", False)):
                raise ValueError("generation_config with do_sample=True is not supported by RequestQueue (greedy decoding only)")
            rp = g.get("repetition_penalty")
            if rp is not None and float(rp) != 1.0:
                raise ValueError("generation_config with repetition_penalty is not supported by RequestQueue")
        if solver not in SOLVERS:
            raise ValueError("solver must be one of %s (got %r)" % (SOLVERS, solver))
        steps = int(steps)
        if not 1 <= steps <= self.model._max_steps:
            raise ValueError("steps %d outside [1, %d] (the model's max_diffusion_steps)" % (steps, self.model._max_steps))
        ids = torch.as_tensor(inputs["input_ids"]).cpu().long()
        ids = ids[None] if ids.dim() == 1 else ids
        if ids.shape[0] != 1:
            raise ValueError("inputs: one script per request (input_ids has %d rows)" % ids.shape[0])
        am = inputs.get("attention_mask") if hasattr(inputs, "get") else None
        am = torch.ones_like(ids) if am is None else torch.as_tensor(am).cpu().long().reshape(ids.shape)
        st = inputs.get("speech_tensors") if hasattr(inputs, "get") else None
        voice = None
        if voice_preset is not None:
            voice_preset = self.model._presets_of(voice_preset, 1)[0]
            sim = inputs.get("speech_input_mask") if hasattr(inputs, "get") else None
            sim = None if sim is None else torch.as_tensor(sim).bool().cpu().reshape(ids.shape)[0][am[0].bool()]
            self.model._check_preset_row(voice_preset, ids[0][am[0].bool()], sim, "the request")
        elif st is not None:
            if self.model._voice is None:
                raise N.VVError("voice-prompt prefill needs the acoustic tokenizer encoder weights, which this checkpoint does not have")
            voice = (st, inputs["speech_masks"], torch.as_tensor(inputs["speech_input_mask"]).bool().cpu().reshape(ids.shape)[0])
        # the limits of generate() (modeling_vibevoice_inference.py:372-373, 402, 421-422) for a batch of one
        L0 = ids.shape[1]
        dc = self.model.config.decoder_config
        mnt = dc.max_position_embeddings - L0 if max_new_tokens is None else int(max_new_tokens)
        max_length = L0 + mnt
        init_len = int(am[0].sum())
        max_steps = min(max_length - L0, int(max_length_times * L0))
        max_step_per_sample = min(max_length - init_len, int(max_length_times * init_len))
        pages = (L0 + max_steps + 2 + 63) // 64 + (max_steps + 2 + 63) // 64
        shared = 0 if voice_preset is None else voice_preset.pages
        pages -= shared
        if pages + shared > self._budget:
            raise ValueError("max_total_tokens: the request needs up to %d KV pages, the pool has %d for requests" % (pages + shared, self._budget))
        rid = self._next_rid
        self._next_rid += 1
        self._wait(_Request(rid, ids[0], am[0].bool(), voice, float(cfg_scale), steps, solver, int(seed), max_length, max_steps,
                            max_step_per_sample, pages, voice_preset, int(priority)))
        return rid

    def _wait(self, req: _Request):
        bisect.insort(self._waiting, req, key=_Request.key)

    def cancel(self, rid: int) -> VibeVoiceGenerationOutput:
        """End request `rid` now (between yields of `run()`), whether it waits, is being admitted, runs or is parked: frees its row and
        KV pages and returns what it produced so far (the prompt and the audio of the frames it ran)."""
        for r, row in enumerate(self._rows):
            if row is not None and row.req.rid == rid:
                return self._finish(r)
        req = next((w for w in self._waiting if w.rid == rid), None)
        if req is None:
            raise KeyError("request %r is not queued or live" % (rid,))
        self._waiting.remove(req)
        row = req.parked
        if row is None:
            return VibeVoiceGenerationOutput(sequences=req.ids[None].clone(), speech_outputs=[None], reach_max_step_sample=torch.tensor([False]))
        self._drop_parked(req)
        with torch.cuda.stream(self.eng.stream):
            audio = torch.cat(row.audio, dim=-1) if row.audio else None
        self.eng.sync()
        return VibeVoiceGenerationOutput(sequences=torch.tensor([row.seq], dtype=torch.long), speech_outputs=[audio],
                                         reach_max_step_sample=torch.tensor([row.reach_max]))

    def _drop_parked(self, req: _Request):
        """release a parked request's pages (its KV records), its host copies and its charge"""
        row = req.parked
        hp, hn = row.park[:2]
        for h in (hp, hn):
            if h is not None:
                self.eng.kv_park_release(h)
        req.parked = None
        if row.host is not None:
            self.host_bytes_used -= row.host_bytes
            row.host, row.host_bytes = None, 0
        else:
            self._pages_used -= req.pages

    @staticmethod
    def _swapped(req: _Request) -> bool:
        return req.parked is not None and req.parked.host is not None

    def _held_rows(self) -> List[_Row]:
        """the rows whose pages are in the pool: live ones and parked ones"""
        return [row for row in self._rows if row is not None] + [w.parked for w in self._waiting if w.parked is not None]

    def _prefixes(self) -> dict:
        """handle -> pages of every shared prefix in the pool (this queue's presets, and any other preset used on the model since)."""
        return getattr(self.eng, "prefix_pages", None) or {}

    def preset_pages(self, extra=None) -> int:
        """KV pages of shared prefixes: every prefix in the pool, the released ones live or parked rows still hold, and the presets that
        live rows build or wait for (+ `extra`'s when it is not in the pool)."""
        held, pending = dict(self._prefixes()), {}
        for row in self._held_rows():
            p = row.req.preset
            if p is None or not p.shared:
                continue
            if row.prefix is not None:
                held[row.prefix] = p.pages
            elif not p.resident():
                pending[id(p)] = p.pages
        if extra is not None and extra.shared and not extra.resident():
            pending[id(extra)] = extra.pages
        return sum(held.values()) + sum(pending.values())

    def _fits(self, req, freed: int = 0) -> bool:
        """whether `req`'s worst case fits beside everything held, less `freed` pages (a parked request holds its shared pages)"""
        extra = req.preset if req.parked is None else None
        return self._pages_used - freed + self.preset_pages(extra) + req.pages <= self._budget

    def _evict(self, req) -> bool:
        """Release shared prefixes until the request at the head fits: first those no live, parked or waiting request uses, then, with
        no row live, every one but its own and those of parked rows (their requests build them again).  Without the second step a pool
        filled by resident presets would keep the head waiting for ever; `submit` made sure it fits beside its own preset alone.  Returns
        whether it fits now."""
        live = any(row is not None for row in self._rows)
        keep = {row.prefix for row in self._held_rows()}
        parked = {w.parked.prefix for w in self._waiting if w.parked is not None}
        own = {req.preset._handle} if req.preset is not None and req.preset.resident() else set()
        used = {w.preset._handle for w in self._waiting if w.preset is not None and w.preset.resident()}
        for spare in ([keep | used | own] if live else [keep | used | own, own | parked]):
            for h in [h for h in self._prefixes() if h not in spare]:
                self.eng.kv_prefix_release(h)
            if self._fits(req):
                return True
        return False

    # ---- the loop ---------------------------------------------------------------------------------------------------------------------
    def run(self) -> Iterator[Tuple[int, VibeVoiceGenerationOutput]]:
        """Serve every queued request (and those submitted while iterating); yields (request id, output) in completion order."""
        eng, model = self.eng, self.model
        if model.model.noise_scheduler is not None and model.model.noise_scheduler is not eng.scheduler:
            eng.set_scheduler(model.model.noise_scheduler)      # as generate() does: the solvers use the installed scheduler's configuration
        eng.codec_state_reset()
        for s in range(2 * self.B):
            eng.kv_set_len(s, 0)
        self._modes = None
        self._start_emb = eng.embed_gather([model._tok.speech_start_id])[0]
        self._set_nmax(max([r.steps for r in self._waiting], default=1))
        try:
            while self._waiting or any(r is not None for r in self._rows):
                done = self._admit()
                self._prefill_progress()
                if any(r is not None and r.step >= 0 for r in self._rows):
                    done += self._frame()
                for item in done:
                    yield item
        finally:
            for s in range(2 * self.B):
                eng.kv_set_len(s, 0)
            for w in [w for w in self._waiting if w.parked is not None]:      # dropped with the live rows when run() is left early
                self._drop_parked(w)
                self._waiting.remove(w)
            self._rows = [None] * self.B
            self._pages_used = 0
            self.host_bytes_used = 0
            eng.set_row_mode([1] * (2 * self.B))
            eng.sampler_per_row(0)
            eng.sync()

    def _set_nmax(self, n: int):
        """Per-row sampler with n steps per frame; re-sets the live rows' settings (switching clears them)."""
        self._nmax = n
        self.eng.sampler_per_row(n)
        for r, row in enumerate(self._rows):
            if row is not None:
                self.eng.set_row_sampler(r, row.req.steps, row.req.solver, row.req.cfg_scale)

    def _admit(self) -> List[Tuple[int, VibeVoiceGenerationOutput]]:
        eng, model, done = self.eng, self.model, []
        while self._waiting:
            req = self._waiting[0]
            if req.max_steps <= 0:                      # generate() runs no step: the prompt comes back as it is
                self._waiting.pop(0)
                done.append((req.rid, VibeVoiceGenerationOutput(sequences=req.ids[None].clone(), speech_outputs=[None],
                                                                reach_max_step_sample=torch.tensor([False]))))
                continue
            free = [r for r in range(self.B) if self._rows[r] is None]
            victim = None if free else self._victim(req)
            if not free and victim is None:
                break
            if (req.parked is None or self._swapped(req)) and not (self._fits(req) or self._evict(req) or self._swap_for(req, victim)):
                # parked requests hold their pages whatever runs: resuming them on rows the head cannot use is how those pages come back
                for w in [w for w in self._waiting if w.parked is not None and not self._swapped(w)][:len(free)]:
                    self._waiting.remove(w)
                    self._resume(w, free.pop(0))
                break
            free = [r for r in range(self.B) if self._rows[r] is None]      # _swap_for may have parked rows, the victim among them
            if not free:
                self._park(victim)
                free = [victim]
            self._waiting.pop(0)
            if req.parked is not None:
                self._resume(req, free[0])
                continue
            self._pages_used += req.pages
            r = free[0]
            if req.steps > self._nmax:
                self._set_nmax(req.steps)
            eng.set_row_sampler(r, req.steps, req.solver, req.cfg_scale)
            row = _Row(req, torch.Generator().manual_seed(req.seed), torch.Generator(device=eng.device).manual_seed(req.seed),
                       self._admitted, seq=req.ids.tolist())
            self._admitted += 1
            with torch.cuda.stream(eng.stream):
                ids = req.ids[req.keep]
                if req.preset is not None:
                    e = model._preset_embeds(req.preset, ids)
                elif self._native:
                    e = eng.embed_gather(ids)
                else:
                    e = model._lm_sd["model.language_model.embed_tokens.weight"][ids.to(eng.device)]
                if req.voice is not None:          # the voice embeddings at the speech positions (_prefill_rows)
                    st, sm, sim = req.voice
                    ve = model._voice(torch.as_tensor(st), torch.as_tensor(sm).bool(), model._scale, model._bias, generator=row.gen_dev)
                    e = e.clone()
                    e[sim[req.keep].to(e.device)] = ve.to(e.device, e.dtype)
            row.embeds = e
            self._rows[r] = row
        return done

    def _victim(self, req: _Request) -> Optional[int]:
        """The row `req` may preempt: among the rows of strictly lower priority that have run a frame, the lowest priority, then the most
        recently admitted; None when there is none."""
        rows = [r for r, row in enumerate(self._rows) if row is not None and row.step >= 1 and row.req.priority < req.priority]
        return min(rows, key=lambda r: (self._rows[r].req.priority, -self._rows[r].order), default=None)

    def _park(self, r: int):
        """Set row r's request aside between frames: both sequences' pages (still charged), its codec state and its next input rows go
        with the `_Row`, which keeps its generators, tokens, step and audio; the request waits again at its own priority and order."""
        eng, B, row = self.eng, self.B, self._rows[r]
        hp = eng.kv_park(r)
        hn = eng.kv_park(B + r) if eng.kv_len(B + r) > 0 else None     # the negative sequence is empty after a <speech_start>
        codec = eng.codec_state_save(r)
        with torch.cuda.stream(eng.stream):
            emb = eng.embeds[[r, B + r]]
        eng.codec_state_zero([r])
        row.park = (hp, hn, codec, emb)
        row.req.parked = row
        self._rows[r] = None
        self.parks += 1
        self._wait(row.req)

    def _swap_for(self, req: _Request, victim: Optional[int]) -> bool:
        """Swap out lower-priority requests until `req` fits the pool (class docstring): plan the shortest run of candidates first, then
        park the running ones among them and swap every one.  Returns whether anything was swapped (then `req` fits)."""
        if self._host_budget <= 0:
            return False
        order = lambda row: (row.req.priority, -row.order)
        parked = sorted((w.parked for w in self._waiting if w.parked is not None and w.parked.host is None and w.priority < req.priority),
                        key=order)
        running = sorted((row for r, row in enumerate(self._rows)
                          if row is not None and r != victim and row.step >= 1 and row.req.priority < req.priority), key=order)
        room, freed, plan = self._host_budget - self.host_bytes_used, 0, []
        for row in ([self._rows[victim]] if victim is not None else []) + parked + running:
            n = self._private_bytes(row)
            if n > room:
                continue
            plan.append(row)
            room -= n
            freed += row.req.pages
            if self._fits(req, freed):
                break
        else:
            return False
        for row in plan:
            if row.park is None:
                self._park(next(r for r, x in enumerate(self._rows) if x is row))
            self._swap_out(row)
        return True

    def _private_bytes(self, row: _Row) -> int:
        """host bytes a swap-out of `row` would take now: its parked records' private pages, or those its sequences would park"""
        eng, B = self.eng, self.B
        if row.park is not None:
            return sum(eng.kv_swap_bytes(h) for h in row.park[:2] if h is not None)
        r = next(r for r, x in enumerate(self._rows) if x is row)
        pages = eng.kv_seq_pages(r) - (row.req.preset.pages if row.prefix is not None else 0)
        if eng.kv_len(B + r) > 0:                       # _park parks the negative sequence only when it holds entries
            pages += eng.kv_seq_pages(B + r)
        return pages * eng.kv_page_bytes

    def _swap_out(self, row: _Row):
        """move parked `row`'s private pages to pinned host memory: its worst case leaves the pool charge, its bytes join the host's"""
        row.host_bytes = self._private_bytes(row)
        row.host = [None if h is None else self.eng.kv_swap_out(h) for h in row.park[:2]]
        self._pages_used -= row.req.pages
        self.host_bytes_used += row.host_bytes
        self.swaps += 1

    def _resume(self, req: _Request, r: int):
        """Continue a parked request on free row r (any index): its pages (copied back first when swapped), codec state, next input
        and sampler settings."""
        eng, B, row = self.eng, self.B, req.parked
        hp, hn, codec, emb = row.park
        if row.host is not None:
            for h, buf in zip((hp, hn), row.host):
                if h is not None:
                    eng.kv_swap_in(h, buf)
            self._pages_used += req.pages
            self.host_bytes_used -= row.host_bytes
            row.host, row.host_bytes = None, 0
        eng.set_row_sampler(r, req.steps, req.solver, req.cfg_scale)
        eng.kv_unpark(hp, r)
        if hn is not None:
            eng.kv_unpark(hn, B + r)
        eng.codec_state_load(r, codec)
        with torch.cuda.stream(eng.stream):
            eng.embeds[r].copy_(emb[0])
            eng.embeds[B + r].copy_(emb[1])
        row.park, req.parked = None, None
        row.order = self._admitted
        self._admitted += 1
        self._rows[r] = row

    def _prefill_progress(self):
        """Prefill the admitting rows, oldest first: whole prompts, or at most max_prefill_tokens_per_frame tokens in all."""
        eng, B = self.eng, self.B
        budget = self._chunk
        for r in sorted((r for r in range(B) if self._rows[r] is not None and self._rows[r].step < 0), key=lambda r: self._rows[r].order):
            row = self._rows[r]
            p = row.req.preset
            if p is not None and p.shared and row.done == 0 and not row.builds:
                if p._attach(r):
                    row.done, row.prefix = p.shared, p._handle
                elif any(o is not None and o.builds and o.req.preset is p for o in self._rows):
                    continue                            # attaches once the row building the preset's pages has made them
                else:
                    row.builds = True
            n_all = row.embeds.shape[0]
            while True:                                 # a row building its preset stops at `shared` once, to make the prefix
                n = (p.shared if row.builds else n_all) - row.done
                if budget is not None:
                    if budget < n:
                        n = budget // 64 * 64           # chunk boundaries on 64-token rows: the native prefill's own chunk grid
                    budget -= n
                if n <= 0:
                    break
                with torch.cuda.stream(eng.stream):
                    if self._native or p is not None:
                        row.hid = eng.lm_prefill(r, row.embeds[row.done:row.done + n], pos0=row.done)
                    else:
                        row.hid = self.model._prefill.run(eng, r, row.embeds)
                row.done += n
                eng.kv_set_len(r, row.done)
                if not (row.builds and row.done == p.shared):
                    break
                p._adopt(r)
                row.builds, row.prefix = False, p._handle
            if n <= 0:
                break
            if row.done < n_all:
                continue
            # step 0 of generate(): the negative sequence restarts at [<speech_start>] (decoded by the next frame's lm_decode, with the
            # positive row switched off there), the first token comes from the prefill's last hidden state
            row.embeds = None
            row.step = 0
            eng.kv_set_len(B + r, 0)
            with torch.cuda.stream(eng.stream):
                eng.embeds[B + r].copy_(self._start_emb)

    def _frame(self) -> List[Tuple[int, VibeVoiceGenerationOutput]]:
        """One step of every running row: the loop body of generate() (modeling.py), rows at their own steps."""
        eng, B, model = self.eng, self.B, self.model
        tok = model._tok
        start_id, end_id, diff_id, eos_id = tok.speech_start_id, tok.speech_end_id, tok.speech_diffusion_id, tok.eos_token_id
        run = [r for r in range(B) if self._rows[r] is not None and self._rows[r].step >= 0]
        fresh = [r for r in run if self._rows[r].step == 0]
        # rows admitting (and free rows) neither read nor append K/V; a row at step 0 decodes only its negative [<speech_start>]
        modes = [0] * (2 * B)
        for r in run:
            modes[r], modes[B + r] = (1 if self._rows[r].step > 0 else 0), 1
        if modes != self._modes:
            eng.set_row_mode(modes)
            self._modes = modes
        eng.lm_decode()
        if fresh:
            with torch.cuda.stream(eng.stream):
                for r in fresh:
                    eng.hidden[r].copy_(self._rows[r].hid)
            eng.lm_head(eng.hidden)                     # the decode's own head kernel: the other rows' tokens do not change
        toks, _ = eng.read_tokens()
        adv = [0] * (2 * B)
        tl = [eos_id] * B
        end_rows, start_rows, diff_rows = [], [], []
        for r in run:
            row = self._rows[r]
            t = int(toks[r])
            row.seq.append(t)
            if t == eos_id:
                row.finished = True
            elif row.step >= row.req.max_step_per_sample:
                row.finished = row.reach_max = True
            if t == end_id:
                end_rows.append(r)
            if not row.finished and t == start_id:
                start_rows.append(r)
            diff = not row.finished and t == diff_id
            adv[r] = 0 if row.step == 0 else 1
            adv[B + r] = 1 if diff else 0
            tl[r] = t
            if diff:
                diff_rows.append(r)
        if end_rows:
            eng.codec_state_zero(end_rows)
        eng.kv_commit(adv)
        for r in start_rows:
            eng.kv_set_len(B + r, 0)
        eng.embed_tokens(tl + tl, eng.embeds)
        if diff_rows:
            vae = model.config.acoustic_vae_dim
            noise = torch.cat([torch.randn(2, vae, generator=self._rows[r].gen_cpu)[:1] for r in diff_rows])
            eng.upload_frame_inputs(noise, diff_rows)
            for r in diff_rows:
                req = self._rows[r].req
                if req.solver == "sde-dpmsolver++":     # one [2, 64] draw per solver step, as the solo run's upload_step_noise
                    with torch.cuda.stream(eng.stream):
                        sn = torch.cat([torch.randn(2, vae, device=eng.device, generator=self._rows[r].gen_dev)[:1]
                                        for _ in range(req.steps)])
                    eng.upload_row_step_noise(r, sn)
            eng.frame_tail(1.0)                          # per-row mode: the CFG scales come from the row settings
            with torch.cuda.stream(eng.stream):
                chunk = eng.audio[diff_rows].clone()
            for i, r in enumerate(diff_rows):
                self._rows[r].audio.append(chunk[i:i + 1])
        done = []
        for r in run:
            row = self._rows[r]
            row.step += 1
            # the checks at the top of generate()'s next iteration
            if row.step < row.req.max_steps and not row.finished:
                if len(row.seq) < row.req.max_length:
                    continue
                row.reach_max = True
            done.append((row.req.rid, self._finish(r)))
        return done

    def _finish(self, r: int) -> VibeVoiceGenerationOutput:
        eng, row = self.eng, self._rows[r]
        eng.sync()
        with torch.cuda.stream(eng.stream):
            audio = torch.cat(row.audio, dim=-1) if row.audio else None
        eng.sync()
        eng.kv_set_len(r, 0)
        eng.kv_set_len(self.B + r, 0)
        eng.codec_state_zero([r])
        self._rows[r] = None
        self._pages_used -= row.req.pages
        return VibeVoiceGenerationOutput(sequences=torch.tensor([row.seq], dtype=torch.long), speech_outputs=[audio],
                                         reach_max_step_sample=torch.tensor([row.reach_max]))


# ---- streaming-0.5B -------------------------------------------------------------------------------------------------------------------
@dataclass
class _StreamRequest:
    rid: int
    prompt: List[int]                   # input_ids when there is no cached prompt: run one token per tick after the negative token
    prefilled: Any                      # all_prefilled_outputs, or None
    neg_id: int
    seq0: List[int]                     # the TTS-LM's view of the prompt: where `sequences` start
    text: List[int]                     # every text token pushed so far
    complete: bool
    cfg_scale: float
    steps: int
    seed: int
    max_length: int
    pages: int                          # worst-case KV pages of the three sequences
    streamer: Any


@dataclass
class _Slot:
    req: _StreamRequest
    gen: torch.Generator                # the request's `randn(2, vae)[:1]` frame noise
    seq: List[int]
    prompt: List[int]                   # prompt tokens still to run; the first one goes to the negative row while `neg_first`
    neg_first: bool
    window: List[int] = field(default_factory=list)     # text tokens of the current window still to run
    taken: int = 0                      # text tokens taken into windows so far
    frames: int = 0                     # speech frames left in the current window
    audio: List[torch.Tensor] = field(default_factory=list)


class StreamingRequestQueue:
    """Continuous batching of streaming-0.5B requests over a `max_slots` model (`streaming.VibeVoiceStreamingForConditionalGenerationInference`).

        q = StreamingRequestQueue(model, max_total_tokens=...)
        rid = q.submit(**inputs, tts_text_ids=first_ids, text_complete=False, cfg_scale=1.5, steps=5, max_new_tokens=600, seed=0,
                       audio_streamer=AudioStreamer(1))
        q.push_text(rid, more_ids, complete=True)       # text may arrive while the request speaks
        done = q.step()                                 # one tick; [(rid, VibeVoiceGenerationOutput)] of the requests that finished
        for rid, out in q.run(): ...                    # or: tick until every request has finished

    Every tick advances each slot by one unit of the solo loop (`streaming.generate`): one prompt token, one text token, or one speech
    frame.  The slots' units share the launches: one lower-stack program for the slots on a text token, one sampler -> acoustic decoder ->
    connector pass for the slots on a speech frame, one type-embedding launch, one upper-stack (TTS-LM) program for all of them (text
    slots on one row, speech slots on both), and one EOS-classifier launch whose read-back is the tick's only host synchronisation.  A
    slot takes its next text window when 5 tokens are pending, or fewer once its text is complete; until then it waits and takes part in
    no launch, so the output does not depend on how the text was split into `push_text` calls.

    A request's output equals `torch.manual_seed(seed); model.set_ddpm_inference_steps(steps); model.generate(<that request with its
    whole text>, cfg_scale=cfg_scale)`: each request has its own CPU generator for the frame noise and its own sampler settings
    (`Engine.set_row_sampler`).  At the EOS decision the slot is freed at once; the solo loop still runs the rest of that speech window,
    whose audio it does not keep, so only its `1` tokens are appended to `sequences` here.  Audio reaches each request's streamer through
    the engine's pinned ring after the tick's read-back.  Driven from one thread; streamers may be read from others."""

    def __init__(self, model, max_total_tokens: int):
        eng = model.engine
        if eng is None or not eng.finalized:
            raise N.VVError("weights not loaded")
        self.model, self.eng, self.S = model, eng, model.max_slots
        eng.kv_init(int(max_total_tokens))
        self._budget = eng.kv_pages - 2 * eng.B            # every decode keeps one page for each sequence's next entry
        self._waiting: Deque[_StreamRequest] = collections.deque()
        self._reqs = {}                                    # rid -> request, until it has finished
        self._slots: List[Optional[_Slot]] = [None] * self.S
        self._next_rid = 0
        self._pages_used = 0
        self._nmax = 0
        self._started = False
        self._pending_audio: List[Tuple[Any, List[int], List[Any]]] = []
        self.last_tick = (0, 0)                            # (slots on a text or prompt token, slots on a speech frame) of the last tick

    # ---- requests ---------------------------------------------------------------------------------------------------------------------
    def submit(self, inputs=None, tts_text_ids=None, text_complete: bool = True, cfg_scale: float = 1.0, steps: Optional[int] = None,
               max_new_tokens: Optional[int] = None, seed: int = 0, audio_streamer=None, solver: str = "dpmsolver++",
               stop_check_fn=None, **kwargs) -> int:
        """Queue one request; takes what `generate()` takes (the processor's output, with or without `all_prefilled_outputs`).  Returns
        the request id that `step()` / `run()` report."""
        model = self.model
        if stop_check_fn is not None:
            raise ValueError("stop_check_fn is not supported by StreamingRequestQueue (use cancel(rid))")
        if solver != "dpmsolver++":
            raise ValueError("solver %r: the streaming loop samples with dpmsolver++ only" % (solver,))
        steps = int(model.ddpm_inference_steps if steps is None else steps)
        if not 1 <= steps <= model._max_steps:
            raise ValueError("steps %d outside [1, %d] (the model's max_diffusion_steps)" % (steps, model._max_steps))
        if audio_streamer is not None and getattr(audio_streamer, "batch_size", 1) != 1:
            raise ValueError("audio_streamer must have batch size 1 (one streamer per request)")
        tokenizer = kwargs.pop("tokenizer", None)
        neg_id = kwargs.pop("neg_text_input_id", None)
        prefilled = kwargs.pop("all_prefilled_outputs", None)
        ids = kwargs["input_ids"] if "input_ids" in kwargs else inputs
        if ids is None:
            raise ValueError("input_ids are required")
        ids = torch.as_tensor(ids).cpu().long()
        if ids.dim() == 2:
            if ids.shape[0] != 1:
                raise ValueError("one request per submit (input_ids has %d rows)" % ids.shape[0])
            ids = ids[0]
        tts_ids = kwargs.get("tts_lm_input_ids")
        tts_ids = ids if tts_ids is None else torch.as_tensor(tts_ids).cpu().long()
        if tts_ids.dim() == 2 and tts_ids.shape[0] != 1:
            raise ValueError("one request per submit (tts_lm_input_ids has %d rows)" % tts_ids.shape[0])
        tts_ids = tts_ids.reshape(-1)
        if prefilled is None and neg_id is None and tokenizer is None:
            raise ValueError("without all_prefilled_outputs the negative prompt needs neg_text_input_id= or tokenizer=")
        neg_id = 0 if prefilled is not None and neg_id is None and tokenizer is None else \
            int(tokenizer.convert_tokens_to_ids("<|image_pad|>") if neg_id is None else neg_id)
        text = [] if tts_text_ids is None else torch.as_tensor(tts_text_ids).cpu().long().reshape(-1).tolist()
        L0 = int(tts_ids.numel())
        mnt = model.config.decoder_config.max_position_embeddings - L0 if max_new_tokens is None else int(max_new_tokens)
        if prefilled is not None:
            lens = [self._cache_len(prefilled[k].past_key_values) for k in ("lm", "tts_lm", "neg_tts_lm")]
        else:
            lens = [int(ids.numel()), int(ids.numel()), 1]
        pages = sum((n + mnt + 2 + 63) // 64 for n in lens)
        if pages > self._budget:
            raise ValueError("max_total_tokens: the request needs up to %d KV pages, the pool has %d for requests" % (pages, self._budget))
        rid = self._next_rid
        self._next_rid += 1
        req = _StreamRequest(rid, [] if prefilled is not None else ids.tolist(), prefilled, neg_id, tts_ids.tolist(), text, bool(text_complete),
                             float(cfg_scale), steps, int(seed), L0 + mnt, pages, audio_streamer)
        self._waiting.append(req)
        self._reqs[rid] = req
        return rid

    @staticmethod
    def _cache_len(cache) -> int:
        if hasattr(cache, "key_cache"):
            return int(cache.key_cache[0].shape[2])
        if hasattr(cache, "layers"):
            return int(next(l.keys for l in cache.layers if getattr(l, "keys", None) is not None).shape[2])
        return int(cache[0][0].shape[2])

    def push_text(self, rid: int, ids, complete: bool = False):
        """Append text token ids to request `rid` (while it waits or speaks); `complete=True` marks its text as whole."""
        req = self._reqs.get(rid)
        if req is None:
            raise KeyError("request %r is not queued or live" % (rid,))
        if req.complete:
            raise ValueError("request %d: its text is already complete" % rid)
        req.text += torch.as_tensor(ids).cpu().long().reshape(-1).tolist()
        req.complete = bool(complete)

    def cancel(self, rid: int) -> VibeVoiceGenerationOutput:
        """End request `rid` now (between ticks): returns what it produced so far and ends its streamer."""
        req = self._reqs.get(rid)
        if req is None:
            raise KeyError("request %r is not queued or live" % (rid,))
        for s, slot in enumerate(self._slots):
            if slot is not None and slot.req is req:
                return self._finish(s, False)
        self._waiting.remove(req)
        del self._reqs[rid]
        if req.streamer is not None:
            req.streamer.end()
        return VibeVoiceGenerationOutput(sequences=torch.tensor([req.seq0], dtype=torch.long), speech_outputs=[None],
                                         reach_max_step_sample=torch.tensor([False]))

    # ---- the loop ---------------------------------------------------------------------------------------------------------------------
    def run(self) -> Iterator[Tuple[int, VibeVoiceGenerationOutput]]:
        """Tick until nothing is queued or live; yields (request id, output) in completion order.  Raises RuntimeError when every live
        request waits for text that is not complete (push_text from inside the loop, or use step())."""
        while self._waiting or any(s is not None for s in self._slots):
            done = self.step()
            if not done and self.last_tick == (0, 0):
                raise RuntimeError("every live request waits for text that is not complete (push_text(..., complete=True))")
            for item in done:
                yield item

    def _start(self):
        eng = self.eng
        eng.codec_state_reset()
        for s in range(2 * eng.B):
            eng.kv_set_len(s, 0)
        with torch.cuda.stream(eng.stream):
            eng.feat.zero_()                               # no semantic branch: the connector adds RMSNorm(0) = 0
            self._hsave = torch.empty_like(eng.hidden)
        self._set_nmax(max([r.steps for r in self._waiting], default=1))
        self._started = True

    def _stop(self):
        eng = self.eng
        eng.set_row_mode([1] * (2 * eng.B))
        eng.sampler_per_row(0)
        eng.sync()
        self._started = False

    def _set_nmax(self, n: int):
        """Per-row sampler with n steps per frame; re-sets the live slots' settings (switching clears them)."""
        self._nmax = n
        self.eng.sampler_per_row(n)
        for s, slot in enumerate(self._slots):
            if slot is not None:
                self.eng.set_row_sampler(s, slot.req.steps, "dpmsolver++", slot.req.cfg_scale)

    def _admit(self):
        eng, model = self.eng, self.model
        while self._waiting:
            req = self._waiting[0]
            free = [s for s in range(self.S) if self._slots[s] is None]
            if not free or self._pages_used + req.pages > self._budget:
                break
            self._waiting.popleft()
            self._pages_used += req.pages
            s = free[0]
            if req.steps > self._nmax:
                self._set_nmax(req.steps)
            eng.set_row_sampler(s, req.steps, "dpmsolver++", req.cfg_scale)
            eng.codec_state_zero([s])
            slot = _Slot(req, torch.Generator().manual_seed(req.seed), list(req.seq0), list(req.prompt), req.prefilled is None)
            if req.prefilled is not None:
                model._import_prefilled(req.prefilled, s)
            self._slots[s] = slot

    def _unit(self, slot: _Slot):
        """The slot's unit of this tick: ("text", token, to_negative_row), ("speech",), ("wait",) or ("max",) (the window exceeds
        max_length: the request ends)."""
        if slot.neg_first:
            return ("text", slot.req.neg_id, True)
        if slot.prompt:
            return ("text", slot.prompt[0], False)
        if slot.window:
            return ("text", slot.window[0], False)
        if slot.frames:
            return ("speech",)
        req = slot.req
        pending = len(req.text) - slot.taken
        if pending < 5 and not req.complete:                                   # TTS_TEXT_WINDOW_SIZE
            return ("wait",)
        cur = req.text[slot.taken:slot.taken + 5]
        slot.taken += len(cur)
        slot.frames = 6                                                        # TTS_SPEECH_WINDOW_SIZE
        if cur:
            slot.seq += cur
            if len(slot.seq) > req.max_length:
                return ("max",)
            slot.window = list(cur)
            return ("text", cur[0], False)
        return ("speech",)

    def step(self) -> List[Tuple[int, VibeVoiceGenerationOutput]]:
        """One tick (see the class docstring); returns [(request id, output)] of the requests that finished in it."""
        eng, model, S = self.eng, self.model, self.S
        if not self._started:
            if not self._waiting:
                self.last_tick = (0, 0)
                return []
            self._start()
        self._admit()
        done = []
        text, speech = [], []                              # slots on a text token: (slot, token, upper row); slots on a speech frame
        for s, slot in enumerate(self._slots):
            if slot is None:
                continue
            u = self._unit(slot)
            if u[0] == "max":
                done.append((slot.req.rid, self._finish(s, True)))
            elif u[0] == "text":
                pos, _, neg = model.slot_rows(s)
                text.append((s, u[1], neg if u[2] else pos))
            elif u[0] == "speech":
                speech.append(s)
        self.last_tick = (len(text), len(speech))
        src, typ, dst, up = [], [], [], []
        if text:                                          # lower stack: the text slots' tokens, output into their `embeds` rows
            toks = [0] * (2 * eng.B)
            for s, t, _ in text:
                toks[model.slot_rows(s)[1]] = int(t)
            rows = [model.slot_rows(s)[1] for s, _, _ in text]
            eng.embed_tokens(toks, eng.embeds)
            eng.set_row_mode(model._mode(rows))
            eng.lm_decode_range(0, model.low, False, out=eng.embeds)
            eng.kv_commit(model._mode(rows))
            for s, _, r in text:
                src.append(model.slot_rows(s)[1])
                typ.append(1)
                dst.append(r)
                up.append(r)
        stepped = []                                       # speech slots that run the TTS-LM step (and the EOS classifier)
        if speech:
            vae = model.config.acoustic_vae_dim
            noise = torch.cat([torch.randn(2, vae, generator=self._slots[s].gen)[:1] for s in speech])
            eng.upload_frame_inputs(noise, speech)
            eng.diffusion_sample(1.0)                      # per-row mode: steps and CFG scales are the slots' own
            eng.codec_decode()
            with torch.cuda.stream(eng.stream):
                chunk = eng.audio[speech].clone()
            streamers = [self._slots[s].req.streamer for s in speech]
            if any(st is not None for st in streamers):
                self._pending_audio.append((eng.stage_audio(speech), list(speech), streamers))
            eng.connect()                                  # -> embeds[s] and embeds[B + s]
            for i, s in enumerate(speech):
                slot = self._slots[s]
                slot.audio.append(chunk[i:i + 1])
                slot.frames -= 1
                slot.seq.append(1)
                if len(slot.seq) > slot.req.max_length:
                    continue
                pos, _, neg = model.slot_rows(s)
                src += [pos, pos]
                typ += [0, 0]
                dst += [pos, neg]
                up += [pos, neg]
                stepped.append(s)
        if up:
            eng.tts_type_embed_rows(eng.embeds, src, typ, dst, eng.embeds)
            # the upper program writes every hidden row: keep the TTS-LM state of the live rows it does not run
            keep = [r for s, slot in enumerate(self._slots) if slot is not None for r in model.slot_rows(s)[::2] if r not in up]
            with torch.cuda.stream(eng.stream):
                for r in keep:
                    self._hsave[r].copy_(eng.hidden[r])
            eng.set_row_mode(model._mode(up))
            eng.lm_decode_range(model.low, model.low + model.tts_layers, True)
            eng.kv_commit(model._mode(up))
            with torch.cuda.stream(eng.stream):
                for r in keep:
                    eng.hidden[r].copy_(self._hsave[r])
        for s, _, _ in text:
            slot = self._slots[s]
            if slot.neg_first:
                slot.neg_first = False
                eng.kv_set_len(model.slot_rows(s)[1], 0)       # the negative prompt's text stack is not used again
            elif slot.prompt:
                slot.prompt.pop(0)
            else:
                slot.window.pop(0)
        probs = eng.eos_probs([model.slot_rows(s)[0] for s in stepped]) if stepped else []
        self._deliver_audio()
        for s in speech:
            slot = self._slots[s]
            if s in stepped:
                if probs[stepped.index(s)] <= 0.5:
                    continue
                for _ in range(slot.frames):               # the rest of the solo loop's window: frames whose audio is not kept
                    slot.seq.append(1)
                    if len(slot.seq) > slot.req.max_length:
                        break
                done.append((slot.req.rid, self._finish(s, False)))
            else:
                done.append((slot.req.rid, self._finish(s, True)))
        if not self._waiting and all(slot is None for slot in self._slots):
            self._stop()
        return done

    def _deliver_audio(self):
        """Hand the staged frames to their streamers (valid after the tick's read-back; otherwise fetch_audio waits for that frame)."""
        for ticket, rows, streamers in self._pending_audio:
            a = self.eng.fetch_audio(ticket)
            for i, st in enumerate(streamers):
                if st is not None:
                    st.put(a[i:i + 1].unsqueeze(1), torch.tensor([0]))
        self._pending_audio = []

    def _finish(self, s: int, reach_max: bool) -> VibeVoiceGenerationOutput:
        eng, slot = self.eng, self._slots[s]
        self._deliver_audio()
        if slot.req.streamer is not None:
            slot.req.streamer.end()
        eng.sync()
        with torch.cuda.stream(eng.stream):
            audio = torch.cat(slot.audio, dim=-1) if slot.audio else None
        eng.sync()
        for r in self.model.slot_rows(s):
            eng.kv_set_len(r, 0)
        eng.codec_state_zero([s])
        self._slots[s] = None
        self._pages_used -= slot.req.pages
        del self._reqs[slot.req.rid]
        return VibeVoiceGenerationOutput(sequences=torch.tensor([slot.seq], dtype=torch.long), speech_outputs=[audio],
                                         reach_max_step_sample=torch.tensor([reach_max]))
