"""Request-level continuous batching over ``engine.SlotDecodeEngine``.

Requests queue FIFO.  Between decode steps the host admits one waiting request into each free slot (a B = 1 prefill into that
slot's cache row, which pauses the other slots for its duration; a prompt of more than ``engine.PREFILL_ROWS`` rows is
prefilled in chunks inside the following decode steps instead, one such prompt at a time, and a long prompt at the head of the
queue waits for the previous one to finish) and every ``sync_every`` steps it reads the device count of
open slots to retire the finished ones and deliver their tokens.  A slot is also retired as soon as the host knows that its
budget is spent.  Each request gets exactly what ``model.generate()`` returns for that request alone: its prompt ids, then the
new tokens up to and including its first EOS, or ``max_new_tokens`` of them.

With ``kv_pages`` the engine is ``engine.PagedSlotDecodeEngine``: the KV cache is a shared pool of 64-position pages, and a
*session* (one conversation) keeps its pages between turns without holding a slot, so each turn prefills only its new suffix,
with exactly what ``generate(past_key_values=...)`` returns for that turn.  At admission a request reserves every page it can
need (its session's pages count towards that), so decoding never runs out of pages and nothing is pre-empted; a request at the
head of the queue that cannot get its pages waits for them (FIFO).  ``PagePool`` is that bookkeeping, on the host alone.
"""
from __future__ import annotations

import collections
import dataclasses
from typing import Callable, Deque, Dict, List, Optional

import torch

from .engine import PREFILL_ROWS, PagedSlotDecodeEngine, SlotDecodeEngine

PAGE = 64       # positions per KV page (ops.PAGE)


def pages_for(positions: int) -> int:
    return -(-int(positions) // PAGE)


@dataclasses.dataclass
class _Session:
    pages: List[int]
    kv_len: int = 0             # positions of the conversation held in its pages
    busy: bool = False          # a turn is queued or running


class PagePool:
    """Host bookkeeping of a pool of ``n_pages`` KV pages shared by requests and sessions (no device state).  A session holds
    the pages of its ``kv_len`` cached positions between turns; a turn (or a request without a session) reserves all the pages
    it can need at admission and gives back, when it retires, every page beyond what its session keeps."""

    def __init__(self, n_pages: int):
        if int(n_pages) < 1:
            raise ValueError(f"the pool needs at least one page, got {n_pages}")
        self.n_pages = int(n_pages)
        self._free: List[int] = list(range(self.n_pages))
        self._sessions: Dict[int, _Session] = {}
        self._next_sid = 0

    @property
    def free_pages(self) -> int:
        return len(self._free)

    def session_pages(self) -> int:
        """Pages held by sessions between turns (not by a running turn beyond its session's share)."""
        return sum(len(s.pages) for s in self._sessions.values())

    def open_session(self) -> int:
        sid = self._next_sid
        self._next_sid += 1
        self._sessions[sid] = _Session([])
        return sid

    def session(self, sid: int) -> _Session:
        s = self._sessions.get(sid)
        if s is None:
            raise KeyError(f"unknown or closed session {sid}")
        return s

    def close_session(self, sid: int) -> None:
        s = self.session(sid)
        if s.busy:
            raise RuntimeError(f"session {sid} has a turn in flight; close it after the turn returns")
        self._free.extend(s.pages)
        del self._sessions[sid]

    def reserve(self, positions: int, sid: Optional[int] = None) -> Optional[List[int]]:
        """The page list of a request that needs ``positions`` positions (its session's pages first), or None (nothing taken)
        when the pool is short."""
        held = self.session(sid).pages if sid is not None else []
        extra = pages_for(positions) - len(held)
        if extra > len(self._free):
            return None
        new = [self._free.pop() for _ in range(max(extra, 0))]
        if sid is not None:
            self._sessions[sid].pages = held + new
            return list(self._sessions[sid].pages)
        return new

    def release(self, pages: List[int], sid: Optional[int] = None, kv_len: int = 0) -> None:
        """A request retired: without a session its pages go back; with one, the session keeps the pages of its first ``kv_len``
        positions and the rest go back."""
        if sid is None:
            self._free.extend(pages)
            return
        s = self.session(sid)
        keep = pages_for(kv_len)
        self._free.extend(s.pages[keep:])
        s.pages, s.kv_len, s.busy = s.pages[:keep], int(kv_len), False


@dataclasses.dataclass
class _Request:
    rid: int
    input_ids: torch.Tensor
    features: dict
    max_new: int
    temperature: float
    top_k: int
    top_p: float
    penalty: float
    u: Optional[torch.Tensor]
    session: Optional[int] = None
    pages: Optional[List[int]] = None
    past: int = 0
    admitted_at: int = -1
    first_token: Optional[torch.cuda.Event] = None


class SlotScheduler:
    """``SlotDecodeEngine(model, slots, max_len, ...)`` plus a FIFO queue.  ``submit`` validates and queues a request and
    returns its id; ``run`` serves until the queue is empty and returns {id: sequence [1, S + n] on the device}.
    ``first_token[id]`` is a CUDA event recorded when the request's first token has been picked (time-to-first-token).

    ``kv_pages``: None keeps the contiguous engine (a ``[max_len]`` cache row per slot); an int makes it
    ``PagedSlotDecodeEngine`` with that many shareable 64-position pages, and enables sessions: ``open_session()`` returns a
    session id, ``submit(..., session=sid)`` queues one turn of that conversation (its prompt must extend the conversation so
    far: the previous turn's prompt, its reply and the new turn's tokens), ``close_session(sid)`` gives its pages back."""

    def __init__(self, model, slots: int = 8, max_len: int = 2048, eos_token_ids=None, pad_token_id: Optional[int] = None,
                 sync_every: int = 8, use_graph: bool = True, kv_pages: Optional[int] = None):
        eos = sorted(set([eos_token_ids] if isinstance(eos_token_ids, int) else (eos_token_ids or [])))
        pad = pad_token_id if pad_token_id is not None else (min(eos) if eos else 0)     # generate()'s default
        if int(sync_every) < 1:
            raise ValueError(f"sync_every must be >= 1, got {sync_every}")
        self.model = model
        self.pool: Optional[PagePool] = None
        if kv_pages is None:
            self.engine = SlotDecodeEngine(model, slots, max_len, eos_token_ids=eos, pad_token_id=pad, use_graph=use_graph)
        else:
            self.engine = PagedSlotDecodeEngine(model, slots, max_len, int(kv_pages), eos_token_ids=eos, pad_token_id=pad,
                                                use_graph=use_graph)
            self.pool = PagePool(int(kv_pages))
        self.sync_every = int(sync_every)
        self.steps = 0
        self.first_token: Dict[int, torch.cuda.Event] = {}
        self._queue: Deque[_Request] = collections.deque()
        self._running: Dict[int, _Request] = {}        # slot -> request
        self._prefilling: Optional[tuple] = None        # (slot, request) of the prompt being prefilled in chunks
        self._next_id = 0
        self._last_poll = 0

    @property
    def capacity(self) -> int:
        return self.engine.max_len

    # -- sessions (paged engine only) -------------------------------------------------------------------------------------------
    def _pool(self) -> PagePool:
        if self.pool is None:
            raise ValueError("sessions need the paged KV cache: SlotScheduler(..., kv_pages=N)")
        return self.pool

    def _session(self, sid: int) -> _Session:
        try:
            return self._pool().session(sid)
        except KeyError:
            raise ValueError(f"unknown or closed session {sid!r}") from None

    def open_session(self) -> int:
        """A new conversation; its turns are submitted with ``session=sid`` and keep their KV cache between turns."""
        return self._pool().open_session()

    def close_session(self, sid: int) -> None:
        """Ends the conversation and gives its pages back to the pool (not while one of its turns is in flight)."""
        if self._session(sid).busy:
            raise RuntimeError(f"session {sid} has a turn in flight; close it after the turn returns")
        self._pool().close_session(sid)

    def session_length(self, sid: int) -> int:
        """Positions of the conversation held in its KV pages: the last turn's sequence minus its last token (not fed yet)."""
        return self._session(sid).kv_len

    @property
    def free_pages(self) -> int:
        return self._pool().free_pages

    def submit(self, features: dict, max_new_tokens: int = 20, do_sample: bool = False, temperature: Optional[float] = None,
               top_k: Optional[int] = None, top_p: Optional[float] = None, repetition_penalty: float = 1.0,
               generator: Optional[torch.Generator] = None, num_beams: int = 1, session: Optional[int] = None) -> int:
        """Queues one request: ``features`` is the processor's output for it (``input_ids`` [1, S] and, for audio, its mel or
        waveform fields).  Arguments and defaults are ``generate()``'s: greedy unless ``do_sample``; sampling defaults to
        temperature 1 and top_k 50; ``top_p`` must lie in [0, 1].  A sampled request draws its uniforms here, as ``generate()``
        does for a batch of one, so a seeded generator gives the same tokens in both.

        ``session``: a turn of that conversation (``open_session``), served like ``generate(past_key_values=...)`` with the
        conversation's cache: ``input_ids`` must extend the ``session_length(sid)`` positions already cached.  One turn per
        session may be in flight.  With a paged engine, a request that needs more pages than the pool has raises ValueError."""
        if num_beams != 1:
            raise NotImplementedError("beam search is not built into the slot engine; use generate(num_beams=...)")
        if top_p is not None and not 0.0 <= float(top_p) <= 1.0:       # NaN fails too
            raise ValueError(f"`top_p` has to be a float in [0, 1], but is {top_p}")
        ids = features.get("input_ids")
        if ids is None or ids.dim() != 2 or ids.shape[0] != 1:
            raise ValueError("submit() takes one request: features['input_ids'] must be [1, S]")
        am = features.get("attention_mask")
        if am is not None and not bool(am.to(torch.bool).all()):
            raise NotImplementedError("a single request has no padding; its attention_mask must be all ones")
        S, n = int(ids.shape[1]), int(max_new_tokens)
        if n < 1:
            raise ValueError(f"max_new_tokens must be >= 1, got {max_new_tokens}")
        if S + n > self.capacity:
            raise ValueError(f"a prompt of {S} tokens plus max_new_tokens={n} exceeds the slot capacity of {self.capacity} positions")
        sess = None
        if session is not None:
            sess = self._session(session)
            if sess.busy:
                raise ValueError(f"session {session} already has a turn in flight")
            if not sess.kv_len < S:
                raise ValueError(f"session {session} holds {sess.kv_len} positions; a turn's prompt of {S} tokens must extend them")
        if self.pool is not None and pages_for(S + n) > self.pool.n_pages:
            raise ValueError(f"a prompt of {S} tokens plus max_new_tokens={n} needs {pages_for(S + n)} KV pages; the pool has "
                             f"{self.pool.n_pages}")
        sampling = bool(do_sample) and (temperature is None or float(temperature) > 0)
        temp = (1.0 if temperature is None else float(temperature)) if sampling else 0.0
        k_top = (50 if top_k is None else int(top_k)) if sampling else 0
        p_top = float(top_p) if sampling and top_p is not None else 1.0
        u = None
        if sampling:
            u = torch.rand(S + n + 1, 1, device=self.engine.pos.device, dtype=torch.float32, generator=generator)
        feats = {k: v for k, v in features.items() if k not in ("input_ids", "attention_mask", "labels")}
        rid = self._next_id
        self._next_id += 1
        self._queue.append(_Request(rid, ids, feats, n, temp, k_top, p_top, float(repetition_penalty or 1.0), u, session))
        if sess is not None:
            sess.busy = True
        return rid

    def _admit(self) -> None:
        eng = self.engine
        dev = eng.pos.device
        for j in range(eng.slots):
            if not self._queue:
                return
            if eng.busy[j]:
                continue
            head = self._queue[0]
            S = int(head.input_ids.shape[1])
            past = self.pool.session(head.session).kv_len if head.session is not None else 0
            long = S - past > PREFILL_ROWS
            if long and self._prefilling is not None:
                return                  # FIFO: it waits until the prompt in flight has been prefilled
            kw = {}
            if self.pool is not None:
                pages = self.pool.reserve(S + head.max_new, head.session)
                if pages is None:
                    return              # FIFO: it waits for pages
                head.pages, head.past = pages, past
                kw = dict(past=past, pages=pages)
            r = self._queue.popleft()
            feats = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in r.features.items()}
            eng.admit(j, r.input_ids, r.max_new, r.temperature, r.top_k, r.top_p, r.penalty, r.u, **kw, **feats)
            r.features, r.u = {}, None
            if long:
                self._prefilling = (j, r)
            else:
                self._started(j, r)

    def _started(self, j: int, r: _Request) -> None:
        """The request's first token has been picked: its budget counts from here."""
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        self.first_token[r.rid] = ev
        r.admitted_at = self.steps
        self._running[j] = r

    def _retire(self, results: Dict[int, torch.Tensor], on_tokens: Optional[Callable]) -> int:
        eng = self.engine
        if int(eng.n_open) >= len(self._running) and not any(self._budget_spent(r) for r in self._running.values()):
            return 0                    # n_open counts the slots still open after the last step: nothing finished
        state = torch.stack([eng.done, eng.cur_len]).cpu()
        freed = 0
        for j in sorted(self._running):
            if not int(state[0, j]):
                continue
            r = self._running.pop(j)
            seq = eng.retire(j, int(state[1, j]))
            if self.pool is not None:   # the conversation keeps every position but the last token, which has not been fed
                self.pool.release(r.pages, r.session, int(state[1, j]) - 1)
            results[r.rid] = seq
            freed += 1
            if on_tokens is not None:
                on_tokens(r.rid, seq)
        return freed

    def _budget_spent(self, r: _Request) -> bool:
        return 1 + self.steps - r.admitted_at >= r.max_new

    def run(self, on_tokens: Optional[Callable[[int, torch.Tensor], None]] = None) -> Dict[int, torch.Tensor]:
        """Serves every queued request; ``on_tokens(id, sequence)`` is called as each one finishes."""
        results: Dict[int, torch.Tensor] = {}
        while self._queue or self._running or self._prefilling is not None:
            self._admit()
            if self._queue and not self._running and self._prefilling is None:
                head = self._queue[0]
                need = pages_for(int(head.input_ids.shape[1]) + head.max_new)
                raise RuntimeError(f"request {head.rid} needs {need} KV pages but only {self.pool.free_pages} of "
                                   f"{self.pool.n_pages} are free: open sessions hold {self.pool.session_pages()}; close some")
            due = any(self._budget_spent(r) for r in self._running.values())
            if due or self.steps - self._last_poll >= self.sync_every:
                self._last_poll = self.steps
                if self._retire(results, on_tokens):
                    continue
                if due:
                    raise RuntimeError("a slot reached its budget on the host but not on the device")
            self.engine.step()
            self.steps += 1
            if self._prefilling is not None and self.engine.prefilling is None:
                j, r = self._prefilling
                self._prefilling = None
                self._started(j, r)
        return results

    def pending(self) -> List[int]:
        pf = [] if self._prefilling is None else [self._prefilling[1].rid]
        return [r.rid for r in self._queue] + pf + [r.rid for r in self._running.values()]
