"""A queue of requests served on one GPU's B rows: a row that finishes takes the next waiting request mid-generation.

A static `generate()` batch runs until its longest row ends, and the frame cost is dominated by the weight stream, not by the number of
live rows, so in a static batch the useful share of the work is mean length / max length.  `RequestQueue` keeps the rows busy instead:

    q = RequestQueue(model, max_total_tokens=...)
    rid = q.submit(inputs, cfg_scale=1.3, steps=10, solver="dpmsolver++", max_new_tokens=None, max_length_times=2, seed=1234)
    for rid, out in q.run():          # VibeVoiceGenerationOutput per request, in completion order
        ...

Each frame runs the per-row loop body of `modeling.generate` (refresh_negative=True) for every live row, each at its own step.  After the
frame the rows that finished are freed (both sequences to length 0, codec state zeroed) and waiting requests are admitted, oldest first,
while the KV pool can hold their worst case.  Sampler settings are per row (`Engine.set_row_sampler`): every row pays the largest step
count of the requests in the queue per frame.

Results do not depend on batch-mates: a request's output equals `torch.manual_seed(seed); model.generate(<that request alone>, ...)` with
`set_ddpm_inference_steps(steps)` and that solver.  Each request has its own CPU generator (diffusion noise, `randn(2, 64)[:1]` per
diffusion frame) and device generator (voice-prompt noise, then SDE step noise), drawn in the solo run's order.
"""
from __future__ import annotations

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
    pages: int                          # worst-case KV pages of both sequences


@dataclass
class _Row:
    req: _Request
    gen_cpu: torch.Generator
    gen_dev: torch.Generator
    order: int                          # admission order (prefill progress goes oldest first)
    embeds: Optional[torch.Tensor] = None   # prompt embeddings while the prefill runs
    done: int = 0                       # prompt tokens prefilled so far
    hid: Optional[torch.Tensor] = None  # final-norm hidden state of the last prompt token
    step: int = -1                      # generation step of the next frame; -1 while admitting
    seq: List[int] = field(default_factory=list)
    finished: bool = False
    reach_max: bool = False
    audio: List[torch.Tensor] = field(default_factory=list)


class RequestQueue:
    """Continuous batching of single-script requests over the model's B rows (see the module docstring).

    `max_total_tokens` sizes the KV pool once, here (re-sizing it later would drop every sequence).  Prompts are prefilled on the model's
    prefill path: `TorchPrefill` when the model keeps one and does not default to the native prefill, else the native prefill
    (`vv_lm_prefill`) -- the token-by-token prefill of `generate()` cannot admit a row while other rows run.  A long prompt stalls every
    other row for its whole prefill; `max_prefill_tokens_per_frame` (native prefill only, rounded down to a multiple of 64) spreads it over
    frames, which is exact because the native prefill gives the same result for any chunking."""

    def __init__(self, model, max_total_tokens: int, max_prefill_tokens_per_frame: Optional[int] = None):
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
        self._waiting: Deque[_Request] = collections.deque()
        self._next_rid = 0
        self._rows: List[Optional[_Row]] = [None] * self.B
        self._pages_used = 0
        self._admitted = 0
        self._nmax = 0
        self._modes: Optional[List[int]] = None

    # ---- requests ---------------------------------------------------------------------------------------------------------------------
    def submit(self, inputs, cfg_scale: float = 1.3, steps: int = 10, solver: str = "dpmsolver++", max_new_tokens: Optional[int] = None,
               max_length_times: float = 2, seed: int = 1234, generation_config=None, logits_processor=None, audio_streamer=None,
               stop_check_fn=None, refresh_negative: bool = True) -> int:
        """Queue one request; `inputs` is the processor output for ONE script (+ its voices).  Returns the request id `run()` reports."""
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
        if st is not None:
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
        if pages > self._budget:
            raise ValueError("max_total_tokens: the request needs up to %d KV pages, the pool has %d for requests" % (pages, self._budget))
        rid = self._next_rid
        self._next_rid += 1
        self._waiting.append(_Request(rid, ids[0], am[0].bool(), voice, float(cfg_scale), steps, solver, int(seed), max_length,
                                      max_steps, max_step_per_sample, pages))
        return rid

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
            self._rows = [None] * self.B
            self._pages_used = 0
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
                self._waiting.popleft()
                done.append((req.rid, VibeVoiceGenerationOutput(sequences=req.ids[None].clone(), speech_outputs=[None],
                                                                reach_max_step_sample=torch.tensor([False]))))
                continue
            free = [r for r in range(self.B) if self._rows[r] is None]
            if not free or self._pages_used + req.pages > self._budget:
                break
            self._waiting.popleft()
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
                if self._native:
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

    def _prefill_progress(self):
        """Prefill the admitting rows, oldest first: whole prompts, or at most max_prefill_tokens_per_frame tokens in all."""
        eng, B = self.eng, self.B
        budget = self._chunk
        for r in sorted((r for r in range(B) if self._rows[r] is not None and self._rows[r].step < 0), key=lambda r: self._rows[r].order):
            row = self._rows[r]
            n_all = row.embeds.shape[0]
            n = n_all - row.done
            if budget is not None:
                if budget < n:
                    n = budget // 64 * 64               # chunk boundaries on 64-token rows: the native prefill's own chunk grid
                budget -= n
            if n <= 0:
                break
            with torch.cuda.stream(eng.stream):
                if self._native:
                    row.hid = eng.lm_prefill(r, row.embeds[row.done:row.done + n], pos0=row.done)
                else:
                    row.hid = self.model._prefill.run(eng, r, row.embeds)
            row.done += n
            eng.kv_set_len(r, row.done)
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
