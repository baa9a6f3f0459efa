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
With ``prefix_cache`` requests that open with the same tokens (a system prompt) also share the pages of that prefix, and
prefill only what follows it.  With ``host_kv_pages`` the pool gets a second tier in pinned host memory: when the head of the
queue cannot get its pages, idle sessions (no turn queued or running) are swapped out to it, least recently used first, and a
swapped-out session's pages come back at its next turn's admission.  Running requests are never swapped.
"""
from __future__ import annotations

import collections
import dataclasses
import numbers
from typing import Callable, Deque, Dict, List, Optional, Sequence, Tuple

import torch

from . import ops
from .constraints import LogitsConstraints
from .stop_strings import StopStrings
from .engine import (PREFILL_ROWS, PagedSlotDecodeEngine, SlotDecodeEngine, TokenLogprobs, check_kv_scales,
                     check_lookup_k)

PAGE = 64       # positions per KV page (ops.PAGE)


def pages_for(positions: int) -> int:
    return -(-int(positions) // PAGE)


@dataclasses.dataclass
class _Session:
    pages: List[int]
    kv_len: int = 0             # positions of the conversation held in its pages
    busy: bool = False          # a turn is queued or running
    host: List[int] = dataclasses.field(default_factory=list)      # swapped out: the host pages of its kv_len positions
    last_used: int = -1         # when its last turn retired (swap-outs take the least recently used first)


class PagePool:
    """Host bookkeeping of a pool of ``n_pages`` KV pages shared by requests and sessions (no device state).  A session holds
    the pages of its ``kv_len`` cached positions between turns; a turn (or a request without a session) reserves all the pages
    it can need at admission and gives back, when it retires, every page beyond what its session keeps.

    Pages are reference-counted, so several requests and sessions can hold one page.  The prefix index (used by
    ``SlotScheduler(prefix_cache=True)``) maps ``(parent, tokens)`` to a page whose K / V hold those 64 token ids right after
    the chain of pages ending at page ``parent`` (None for the first page).  The parent's page id stands for its whole chain
    of token ids: eviction takes a page's indexed descendants with it, so an id never names two chains.  Keys are exact tuples,
    not digests, so no other prompt's K / V can be served.  An indexed page nobody holds is *reclaimable*: it keeps its
    contents and can still be hit, until a reservation that finds no free page evicts it (least recently released first).
    A holder of an indexed page holds its whole chain from the first page, so a page nobody holds has no held descendant.

    ``host_pages`` > 0 adds a host tier of that many pages.  A session then lives on exactly one side: on the device, holding
    device pages as above, or on the host (``swap_out``), holding ``pages_for(kv_len)`` host pages of its own and no device
    pages.  Its next reservation takes every page new and gives the host pages back (``reserve``).  ``swap_candidates`` is the
    policy that picks sessions to swap out."""

    def __init__(self, n_pages: int, host_pages: int = 0):
        if int(n_pages) < 1:
            raise ValueError(f"the pool needs at least one page, got {n_pages}")
        if int(host_pages) < 0:
            raise ValueError(f"the host tier cannot have {host_pages} pages")
        self.n_pages = int(n_pages)
        self.host_pages = int(host_pages)
        self._host_free: List[int] = list(range(self.host_pages))
        self._clock = 0                                 # counts retired session turns (LRU)
        self._free: List[int] = list(range(self.n_pages))
        self._refs: List[int] = [0] * self.n_pages
        self._reclaimable: "collections.OrderedDict[int, None]" = collections.OrderedDict()    # oldest first
        self._index: Dict[tuple, int] = {}              # (parent page or None, 64 token ids) -> page
        self._key: Dict[int, tuple] = {}                # indexed page -> its key
        self._children: Dict[int, set] = {}             # indexed page -> the indexed pages keyed under it
        self._sessions: Dict[int, _Session] = {}
        self._next_sid = 0
        self.evicted = 0                                # cached pages evicted so far

    @property
    def free_pages(self) -> int:
        """Pages a reservation can take now: free ones and reclaimable cached ones."""
        return len(self._free) + len(self._reclaimable)

    @property
    def cached_pages(self) -> int:
        """Pages in the prefix index (held or reclaimable)."""
        return len(self._index)

    @property
    def host_free_pages(self) -> int:
        """Host pages not holding a swapped-out session."""
        return len(self._host_free)

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
        self._drop(s.pages)
        self._host_free.extend(s.host)
        del self._sessions[sid]

    def match(self, page_tokens: Sequence[tuple]) -> List[int]:
        """The indexed pages holding ``page_tokens[0]``, ``page_tokens[1]``, ... (64 token ids each) from position 0 on, as far
        as they match.  Takes nothing."""
        chain, parent = [], None
        for t in page_tokens:
            p = self._index.get((parent, t))
            if p is None:
                break
            chain.append(p)
            parent = p
        return chain

    def reserve(self, positions: int, sid: Optional[int] = None, shared: Sequence[int] = ()) -> Optional[List[int]]:
        """The page list of a request that needs ``positions`` positions (its session's pages first, or the cached pages
        ``shared`` from ``match``, then new ones), or None (nothing taken) when the pool is short.  New pages come from the
        free list first, then by evicting reclaimable cached pages, least recently released first.

        A session on the host holds no device pages, so all of its pages are new; the reservation brings it back to the
        device and frees its host pages.  The caller reads ``session(sid).host`` first and copies those host pages into the
        first ``len(host)`` pages returned before anything else on the stream can write them."""
        held = self.session(sid).pages if sid is not None else []
        shared = list(shared)
        if shared and held:
            raise ValueError("a session that holds pages extends its own; only its first turn can share cached pages")
        if self.shortfall(positions, sid, shared):
            return None
        extra = max(pages_for(positions) - len(held) - len(shared), 0)
        for p in shared:                # held first, so the evictions below cannot take them
            self._acquire(p)
        new = [self._take() for _ in range(extra)]
        pages = held + shared + new
        if sid is not None:
            s = self._sessions[sid]
            s.pages = pages
            self._host_free.extend(s.host)
            s.host = []
            return list(pages)
        return pages

    def shortfall(self, positions: int, sid: Optional[int] = None, shared: Sequence[int] = ()) -> int:
        """How many more device pages ``reserve(positions, sid, shared)`` needs than it can take now (0: it succeeds)."""
        held = self.session(sid).pages if sid is not None else []
        extra = max(pages_for(positions) - len(held) - len(shared), 0)
        return max(extra - (self.free_pages - sum(p in self._reclaimable for p in shared)), 0)

    def swap_candidates(self, need: int, exclude: Optional[int] = None, keep: Sequence[int] = ()) -> Optional[List[int]]:
        """The idle sessions to swap out so that ``need`` more device pages become free, or None when no choice does (then
        nothing should move).  Idle means on the device, no turn queued or running and at least one page held; ``exclude``
        (the waiting request's own session) is never picked.  Sessions are taken least recently used first until the pages
        their swap-out would free - those nobody else holds, other than the pages in ``keep`` (the waiting request's cached
        prefix, which it takes itself) - cover ``need``; None if they never do, or if the host tier cannot hold them all."""
        idle = sorted((s.last_used, sid) for sid, s in self._sessions.items() if sid != exclude and not s.busy and s.pages)
        keep, refs = set(keep), {}
        chosen, freed, host = [], 0, 0
        for _, sid in idle:
            pages = self._sessions[sid].pages
            host += len(pages)
            if host > len(self._host_free):
                return None
            chosen.append(sid)
            for p in pages:
                refs[p] = refs.get(p, self._refs[p]) - 1
                freed += refs[p] == 0 and p not in keep
            if freed >= need:
                return chosen
        return None

    def swap_out(self, sid: int) -> Tuple[List[int], List[int]]:
        """Moves an idle session to the host tier: returns (its device pages, the host pages they must be copied to), and
        drops its device references (shared pages stay with their other holders or become reclaimable).  The caller launches
        that copy before anything else on the stream can write those device pages.  ([], []) if it holds no device pages."""
        s = self.session(sid)
        if s.busy:
            raise ValueError(f"session {sid} has a turn in flight; only idle sessions are swapped out")
        if not s.pages:
            return [], []
        if len(s.pages) > len(self._host_free):
            raise ValueError(f"session {sid} holds {len(s.pages)} pages; the host tier has {len(self._host_free)} free")
        dev, host = s.pages, [self._host_free.pop() for _ in s.pages]
        self._drop(dev)
        s.pages, s.host = [], host
        return dev, host

    def register(self, pages: Sequence[int], page_tokens: Sequence[tuple]) -> None:
        """Indexes ``pages[k]`` under ``page_tokens[k]`` for k = 0, 1, ..., once the holder has written their K / V.  Pages
        that are already indexed under those tokens (the shared part of ``pages``) are passed; the first key that another page
        already holds ends the chain, and the rest of ``pages`` stay private (the first registration wins)."""
        parent = None
        for p, t in zip(pages, page_tokens):
            key = (parent, t)
            if self._key.get(p) != key:
                if key in self._index or p in self._key:
                    return
                if self._refs[p] < 1:
                    raise ValueError(f"page {p} is not held; only a holder can register it")
                self._index[key], self._key[p] = p, key
                if parent is not None:
                    self._children.setdefault(parent, set()).add(p)
            parent = p

    def release(self, pages: List[int], sid: Optional[int] = None, kv_len: int = 0) -> None:
        """A request retired: without a session its pages go back; with one, the session keeps the pages of its first ``kv_len``
        positions and the rest go back.  A page goes back to the free list when nobody holds it, unless it is cached: then it
        becomes reclaimable."""
        if sid is None:
            self._drop(pages)
            return
        s = self.session(sid)
        keep = pages_for(kv_len)
        self._drop(s.pages[keep:])
        s.pages, s.kv_len, s.busy = s.pages[:keep], int(kv_len), False
        s.last_used, self._clock = self._clock, self._clock + 1

    def _acquire(self, p: int) -> None:
        if self._refs[p] == 0:
            del self._reclaimable[p]
        self._refs[p] += 1

    def _take(self) -> int:
        if not self._free:
            self._evict(next(iter(self._reclaimable)))
        p = self._free.pop()
        self._refs[p] = 1
        return p

    def _drop(self, pages: Sequence[int]) -> None:
        for p in reversed(pages):       # last page first, so a chain's tail is evicted before its head
            self._refs[p] -= 1
            if self._refs[p] == 0:
                if p in self._key:
                    self._reclaimable[p] = None
                else:
                    self._free.append(p)

    def _evict(self, p: int) -> None:
        """Unindexes reclaimable page ``p`` and its descendants (unreachable without it) and frees them all."""
        key = self._key.pop(p)
        del self._index[key]
        del self._reclaimable[p]
        if key[0] in self._children:    # not when the parent is being evicted itself
            self._children[key[0]].discard(p)
        for c in self._children.pop(p, ()):
            self._evict(c)
        self._free.append(p)
        self.evicted += 1


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
    prefix: Tuple[tuple, ...] = ()     # token ids of its shareable pages (prefix cache on)
    pages: Optional[List[int]] = None
    past: int = 0
    admitted_at: int = -1
    first_token: Optional[torch.cuda.Event] = None
    logprobs: Optional[int] = None     # alternatives per token asked for (None: no log-probs)
    lookup: Optional[tuple] = None     # (k, n) of prompt lookup (None: the engine has none)
    constraints: Optional[LogitsConstraints] = None
    cutoffs: Optional[tuple] = None    # (min_p, typical_p, epsilon, eta) when sampled with one on
    stop: Optional[StopStrings] = None


class SlotScheduler:
    """``SlotDecodeEngine(model, slots, max_len, ...)`` plus a FIFO queue.  ``submit`` validates and queues a request and
    returns its id; ``run`` serves until the queue is empty and returns {id: sequence [1, S + n] on the device}.
    ``first_token[id]`` is a CUDA event recorded when the request's first token has been picked (time-to-first-token).

    ``kv_pages``: None keeps the contiguous engine (a ``[max_len]`` cache row per slot); an int makes it
    ``PagedSlotDecodeEngine`` with that many shareable 64-position pages, and enables sessions: ``open_session()`` returns a
    session id, ``submit(..., session=sid)`` queues one turn of that conversation (its prompt must extend the conversation so
    far: the previous turn's prompt, its reply and the new turn's tokens), ``close_session(sid)`` gives its pages back.

    ``prefix_cache`` (needs ``kv_pages``): requests that start with the same tokens share the K / V pages of that prefix
    instead of prefilling it again.  A request without a session, or a session's first turn, registers its *shareable* pages
    (the full pages before its first audio row) once their K / V are written; a later such request takes the longest matching
    chain of them, up to its own first audio row and S - 1 positions, and prefills only the rest, as
    ``generate(past_key_values=...)`` with those pages as the cache.  ``cached_tokens[id]`` is the number of positions a request
    took from the cache.  Pages nobody holds stay cached until the pool needs them (least recently released first).  Off by
    default because a hit's bits depend on which earlier request computed the shared K / V: its prefill's row count picked
    its GEMM tiling, so a request can get different bits than when it prefills its whole prompt.

    ``max_logprobs`` (0..20): requests may ask for per-token log-probabilities with ``submit(..., logprobs=k)``, k <=
    ``max_logprobs``.  When such a request finishes, ``logprobs[id]`` holds its ``TokenLogprobs`` (filled before ``on_tokens``
    is called): the chosen tokens' log-probs and their k most likely alternatives, one entry per new token, under the model's
    raw distribution - the log_softmax of the logits before the repetition penalty, temperature, top-k and top-p, as
    OpenAI-style ``logprobs`` report them.  (``generate(output_scores=True)`` gives the processed distribution instead.)  With
    0, the default, the engine allocates nothing for them and its step is unchanged.

    ``kv_cache_dtype`` (needs ``kv_pages`` for ``"fp8_e4m3"``): ``"bf16"`` (the default) or ``"fp8_e4m3"``, a pool of
    ``float8_e4m3fn`` pages that cost half the bytes of bf16 ones, so the same memory holds twice the positions.
    ``kv_scales`` [num_hidden_layers, 2] (positive, finite; default all 1) are each layer's K and V scales.  Every K / V value
    written into the pool is stored as q = e4m3(x / s) (round to nearest even, saturating at +-448, NaN kept) and read back as
    bf16(q * s).  A step's attention therefore sees the dequantized keys, the row's just-appended key included; a B = 1
    admission prefills its new suffix over its own bf16 K / V (as ``generate(past_key_values=...)`` with the dequantized past
    does) and only the pages it writes are quantized.  Sessions, the prefix cache, chunked prefill, sampling, the repetition
    penalty and log-probs work unchanged.

    ``host_kv_pages`` (needs ``kv_pages``; default 0, none): that many pages of pinned host memory (same page size and dtype as
    the pool) form a second tier for idle sessions - conversations with no turn queued or running.  When the request at the
    head of the queue cannot get its pages from free or reclaimable cached ones, idle sessions other than its own are swapped
    out, least recently used first (by when their last turn retired): all of their pages, shared prefix pages included, are
    copied to host pages and their device references dropped.  That happens only if the device pages it would free cover what
    the head lacks and the host tier has room; otherwise nothing moves and the head waits as before.  A swapped-out session's
    next turn reserves every page new, its first ``pages_for(kv_len)`` pages are copied back from the host before its suffix
    is prefilled, and its host pages are freed: the restored pages are private (no longer shared with the prefix cache).  The
    bits of every turn are those of the same workload on a pool large enough never to swap.  ``offload_session(sid)`` swaps a
    session out on request, ``session_on_host(sid)`` tells where it is, ``host_free_pages`` counts the free host pages and
    ``swapped_out_pages`` / ``swapped_in_pages`` the pages moved so far.  Each move is one ``uvx_kv_pages_move`` launch on the
    scheduler's stream (the SMs read or write the host pages over PCIe) between decode steps; it pauses the other slots for
    its duration, as an admission's prefill does.  Running requests are never swapped.

    ``prompt_lookup_num_tokens`` = K (None, the default: off): prompt lookup decoding inside the slot step, up to K drafted
    tokens per slot per step (1 <= K <= 31 and slots * (K + 1) <= 256 rows, else ValueError).  ``submit(...,
    prompt_lookup_num_tokens=k, max_matching_ngram_size=n)`` sets a request's k (None: K, 0: no drafts) and n (None: 2), with
    ``generate()``'s meanings.  A request's tokens, log-probs and kept K / V are those plain slot decoding gives it; a step
    yields 1 to k + 1 of them.  Drafts are taken from the request's own prompt and reply (the leftmost earlier match of its
    last n-gram, sizes n down to 1), so they pay off where a reply repeats its input.  ``accepted_drafts[id]`` is the number
    of drafted tokens the request accepted, filled when it finishes.  While a chunked prompt is in flight every slot decodes
    one token per step; the lookup step's linears run at slots * (K + 1) rows (DESIGN.md §6 has their cost).

    ``max_constraint_tokens`` = N (None, the default: off): requests may take ``generate()``'s token constraints,
    ``submit(..., no_repeat_ngram_size=, min_new_tokens=, min_length=, bad_words_ids=, sequence_bias=, suppress_tokens=,
    begin_suppress_tokens=)``, with its meanings and checks, over the request's whole sequence (a session turn's prompt holds
    the conversation so far).  A request's packed table may hold up to N token ids (each entry's ids; EOS ids count once per
    entry under ``min_*``).  Each slot's settings live in device arrays, so the steps stay captured once; the constraints run
    inside every pick, before the penalty, and a request's tokens are those ``generate()`` gives it alone with the same
    options.  With None the engine allocates nothing for them and its steps are unchanged.

    ``max_stop_table`` = N (None, the default: off): requests may take ``generate()``'s stop strings, ``submit(...,
    stop_strings=, tokenizer=)``, with its meaning and checks.  Each slot holds a packed table of up to N int32 words on the
    device (``StopStrings.n_words`` reports a request's size), written at admission; the check runs inside every pick (the
    plain, mixed, admission and lookup steps), and a slot whose text ends with a stop string finishes as on an EOS id.  With
    None nothing is allocated and the steps are unchanged."""

    def __init__(self, model, slots: int = 8, max_len: int = 2048, eos_token_ids=None, pad_token_id: Optional[int] = None,
                 sync_every: int = 8, use_graph: bool = True, kv_pages: Optional[int] = None, prefix_cache: bool = False,
                 max_logprobs: int = 0, kv_cache_dtype: str = "bf16", kv_scales=None, host_kv_pages: int = 0,
                 prompt_lookup_num_tokens: Optional[int] = None, max_constraint_tokens: Optional[int] = None,
                 max_stop_table: Optional[int] = None):
        eos = sorted(set([eos_token_ids] if isinstance(eos_token_ids, int) else (eos_token_ids or [])))
        pad = pad_token_id if pad_token_id is not None else (min(eos) if eos else 0)     # generate()'s default
        if int(sync_every) < 1:
            raise ValueError(f"sync_every must be >= 1, got {sync_every}")
        if prefix_cache and kv_pages is None:
            raise ValueError("prefix_cache shares KV pages between requests: it needs the paged cache (kv_pages=N)")
        if kv_cache_dtype not in ("bf16", "fp8_e4m3"):
            raise ValueError(f"kv_cache_dtype must be 'bf16' or 'fp8_e4m3', got {kv_cache_dtype!r}")
        if isinstance(host_kv_pages, bool) or not isinstance(host_kv_pages, numbers.Integral) or host_kv_pages < 0:
            raise ValueError(f"host_kv_pages must be an integer >= 0, got {host_kv_pages!r}")
        if host_kv_pages and kv_pages is None:
            raise ValueError("host_kv_pages swaps sessions' KV pages to the host: it needs the paged cache (kv_pages=N)")
        kv = {}
        if kv_cache_dtype == "fp8_e4m3":
            if kv_pages is None:
                raise ValueError("kv_cache_dtype='fp8_e4m3' is a paged pool: it needs kv_pages=N")
            kv = dict(kv_cache_dtype=kv_cache_dtype,
                      kv_scales=check_kv_scales(kv_scales, model.config.text_config.num_hidden_layers))
        elif kv_scales is not None:
            raise ValueError("kv_scales are for kv_cache_dtype='fp8_e4m3'")
        self.prefix_cache = bool(prefix_cache)
        self.cached_tokens: Dict[int, int] = {}
        self.logprobs: Dict[int, TokenLogprobs] = {}
        self.model = model
        self.pool: Optional[PagePool] = None
        lp = {} if max_logprobs == 0 else dict(max_logprobs=max_logprobs)     # the engine validates it
        self.lookup_k = check_lookup_k(int(slots), prompt_lookup_num_tokens)     # 0: off
        if self.lookup_k:
            lp["prompt_lookup_num_tokens"] = self.lookup_k
        if max_constraint_tokens is not None:
            lp["max_constraint_tokens"] = max_constraint_tokens       # the engine validates it
        if max_stop_table is not None:
            lp["max_stop_table"] = max_stop_table                     # the engine validates it
        self._eos = eos
        self.accepted_drafts: Dict[int, int] = {}
        if host_kv_pages:
            kv["host_kv_pages"] = int(host_kv_pages)
        if kv_pages is None:
            self.engine = SlotDecodeEngine(model, slots, max_len, eos_token_ids=eos, pad_token_id=pad, use_graph=use_graph,
                                           **lp)
        else:
            self.engine = PagedSlotDecodeEngine(model, slots, max_len, int(kv_pages), eos_token_ids=eos, pad_token_id=pad,
                                                use_graph=use_graph, **lp, **kv)
            self.pool = PagePool(int(kv_pages), int(host_kv_pages))
        self.swapped_out_pages = 0
        self.swapped_in_pages = 0
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

    def offload_session(self, sid: int) -> None:
        """Swaps an idle session's pages out to the host tier now (a no-op if it is there already or holds no pages); its next
        turn brings them back.  ValueError without a host tier, while a turn of it is queued or running, or when the host tier
        has too few free pages."""
        s = self._session(sid)
        if not self.pool.host_pages:
            raise ValueError("offload_session needs a host tier: SlotScheduler(..., kv_pages=N, host_kv_pages=M)")
        if s.busy:
            raise ValueError(f"session {sid} has a turn in flight; only idle sessions are swapped out")
        self._swap_out(sid)

    def session_on_host(self, sid: int) -> bool:
        """Whether the session's pages are on the host tier (swapped out) rather than in the device pool."""
        return bool(self._session(sid).host)

    def _swap_out(self, sid: int) -> None:
        dev, host = self.pool.swap_out(sid)
        if dev:                         # launched before any later admission or step can write the freed device pages
            self.engine.swap_out(dev, host)
            self.swapped_out_pages += len(dev)

    def session_length(self, sid: int) -> int:
        """Positions of the conversation held in its KV pages: the last turn's sequence minus its last token (not fed yet)."""
        return self._session(sid).kv_len

    @property
    def free_pages(self) -> int:
        """Pages a request can take now (free ones and cached ones nobody holds)."""
        return self._pool().free_pages

    @property
    def cached_pages(self) -> int:
        """Pages in the prefix cache, held or not."""
        return self._pool().cached_pages

    @property
    def host_free_pages(self) -> int:
        """Pages of the host tier not holding a swapped-out session."""
        return self._pool().host_free_pages

    def submit(self, features: dict, max_new_tokens: int = 20, do_sample: bool = False, temperature: Optional[float] = None,
               top_k: Optional[int] = None, top_p: Optional[float] = None, repetition_penalty: float = 1.0,
               generator: Optional[torch.Generator] = None, num_beams: int = 1, session: Optional[int] = None,
               logprobs: Optional[int] = None, prompt_lookup_num_tokens: Optional[int] = None,
               max_matching_ngram_size: Optional[int] = None, no_repeat_ngram_size: Optional[int] = None,
               min_new_tokens: Optional[int] = None, min_length: Optional[int] = None, bad_words_ids=None, sequence_bias=None,
               suppress_tokens=None, begin_suppress_tokens=None, min_p: Optional[float] = None,
               typical_p: Optional[float] = None, epsilon_cutoff: Optional[float] = None,
               eta_cutoff: Optional[float] = None, stop_strings=None, tokenizer=None) -> int:
        """Queues one request: ``features`` is the processor's output for it (``input_ids`` [1, S] and, for audio, its mel or
        waveform fields).  Arguments and defaults are ``generate()``'s: greedy unless ``do_sample``; sampling defaults to
        temperature 1 and top_k 50; ``top_p`` must lie in [0, 1].  A sampled request draws its uniforms here, as ``generate()``
        does for a batch of one, so a seeded generator gives the same tokens in both.

        ``session``: a turn of that conversation (``open_session``), served like ``generate(past_key_values=...)`` with the
        conversation's cache: ``input_ids`` must extend the ``session_length(sid)`` positions already cached.  One turn per
        session may be in flight.  With a paged engine, a request that needs more pages than the pool has raises ValueError.

        ``logprobs``: None records nothing; 0 the log-prob of each chosen token; 1..``max_logprobs`` also that many most likely
        alternatives per token (``logprobs[id]`` once it has finished).  Anything else raises ValueError.

        ``prompt_lookup_num_tokens`` / ``max_matching_ngram_size`` (a scheduler built with ``prompt_lookup_num_tokens``): the
        request's drafts per step, None for the scheduler's K, 0 for none, at most K; its n-gram size, None for 2.

        ``no_repeat_ngram_size``, ``min_new_tokens``, ``min_length``, ``bad_words_ids``, ``sequence_bias``, ``suppress_tokens``,
        ``begin_suppress_tokens`` (a scheduler built with ``max_constraint_tokens``): ``generate()``'s token constraints and
        checks.  ValueError when the scheduler has no constraints or the request's table needs more than
        ``max_constraint_tokens`` ids.

        ``min_p``, ``typical_p``, ``epsilon_cutoff``, ``eta_cutoff``: ``generate()``'s sampling cut-offs and checks, held per
        slot and read by the captured step; ignored when not sampling.

        ``stop_strings`` with ``tokenizer`` (a scheduler built with ``max_stop_table``): ``generate()``'s stop strings and checks.
        ValueError when the scheduler has no stop tables or the request's table needs more than ``max_stop_table`` words."""
        if logprobs is not None:
            self.engine.check_logprobs(logprobs)
        lookup = self._check_lookup(prompt_lookup_num_tokens, max_matching_ngram_size)
        if num_beams != 1:
            raise NotImplementedError("beam search is not built into the slot engine; use generate(num_beams=...)")
        if top_p is not None and not 0.0 <= float(top_p) <= 1.0:       # NaN fails too
            raise ValueError(f"`top_p` has to be a float in [0, 1], but is {top_p}")
        cutoffs = ops.sampling_cutoffs(min_p, typical_p, epsilon_cutoff, eta_cutoff)
        ids = features.get("input_ids")
        if ids is None or ids.dim() != 2 or ids.shape[0] != 1:
            raise ValueError("submit() takes one request: features['input_ids'] must be [1, S]")
        am = features.get("attention_mask")
        if am is not None and not bool(am.to(torch.bool).all()):
            raise NotImplementedError("a single request has no padding; its attention_mask must be all ones")
        S, n = int(ids.shape[1]), int(max_new_tokens)
        ck_args = (no_repeat_ngram_size, bad_words_ids, sequence_bias, min_length, min_new_tokens, suppress_tokens,
                   begin_suppress_tokens)
        cons = None
        if any(a is not None for a in ck_args):
            if self.engine.max_constraint_tokens is None:
                raise ValueError("token constraints need a table per slot: SlotScheduler(..., max_constraint_tokens=N)")
            cons = LogitsConstraints.build(self.model.language_model.lm_head.weight.shape[0], self._eos, S, *ck_args)
            self.engine.check_constraints(cons)
        stop = StopStrings.build(tokenizer, stop_strings)
        if stop is not None:
            if self.engine.max_stop_table is None:
                raise ValueError("stop strings need a table per slot: SlotScheduler(..., max_stop_table=N)")
            self.engine.check_stop(stop)
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
        prefix = ()
        if self.prefix_cache and (sess is None or sess.kv_len == 0):
            # audio rows hold the same placeholder id in every request, so only the full pages before the first one can be keyed
            starts = feats.get("audio_token_start_idx")
            first = min(S, int(starts.min())) if starts is not None and starts.numel() else S
            head = ids[0, :first // PAGE * PAGE].tolist()
            prefix = tuple(tuple(head[i:i + PAGE]) for i in range(0, len(head), PAGE))
        rid = self._next_id
        self._next_id += 1
        self._queue.append(_Request(rid, ids, feats, n, temp, k_top, p_top, float(repetition_penalty or 1.0), u, session,
                                    prefix, logprobs=None if logprobs is None else int(logprobs), lookup=lookup,
                                    constraints=cons, cutoffs=cutoffs if sampling and ops.cutoffs_on(cutoffs) else None,
                                    stop=stop))
        if sess is not None:
            sess.busy = True
        return rid

    def _check_lookup(self, k, n) -> Optional[tuple]:
        """A request's (k, n) of prompt lookup (None when the engine has none), with ``generate()``'s checks."""
        K = self.lookup_k
        if not K:
            if k is not None or n is not None:
                raise ValueError("prompt lookup is set per scheduler: SlotScheduler(..., prompt_lookup_num_tokens=K)")
            return None
        k = K if k is None else k
        if isinstance(k, bool) or not isinstance(k, int) or not 0 <= k <= ops.LOOKUP_MAX_K:
            raise ValueError(f"prompt_lookup_num_tokens must be an integer in [1, {ops.LOOKUP_MAX_K}] (k + 1 rows of the decode "
                             f"step), or 0 for no drafts, got {k!r}")
        if k > K:
            raise ValueError(f"prompt_lookup_num_tokens = {k} exceeds the scheduler's prompt_lookup_num_tokens = {K}")
        n = 2 if n is None else n
        if isinstance(n, bool) or not isinstance(n, int) or n < 1:
            raise ValueError(f"max_matching_ngram_size must be an integer >= 1, got {n!r}")
        return k, n

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
            shared = []
            if head.prefix:             # at least one row (the last) is prefilled: it gives the first token's logits
                shared = self.pool.match(head.prefix[:(S - 1) // PAGE])
                past = PAGE * len(shared)
            long = S - past > PREFILL_ROWS
            if long and self._prefilling is not None:
                return                  # FIFO: it waits until the prompt in flight has been prefilled
            kw = {}
            if self.pool is not None:
                need = S + head.max_new
                short = self.pool.shortfall(need, head.session, shared) if self.pool.host_pages else 0
                if short:               # after free and reclaimable pages, before waiting: swap idle sessions out
                    for sid in self.pool.swap_candidates(short, head.session, shared) or ():
                        self._swap_out(sid)
                restore = self.pool.session(head.session).host if head.session is not None else []
                pages = self.pool.reserve(need, head.session, shared)
                if pages is None:
                    return              # FIFO: it waits for pages
                if restore:             # before the prefill reads them; the freed host pages are rewritten only after this
                    self.engine.swap_in(restore, pages[:len(restore)])
                    self.swapped_in_pages += len(restore)
                head.pages, head.past = pages, past
                kw = dict(past=past, pages=pages)
            r = self._queue.popleft()
            if self.prefix_cache:
                self.cached_tokens[r.rid] = PAGE * len(shared)
            feats = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in r.features.items()}
            if r.logprobs is not None:
                kw["logprobs"] = r.logprobs
            if r.lookup is not None:
                kw["lookup"] = r.lookup
            if r.constraints is not None:
                kw["constraints"] = r.constraints
            if r.cutoffs is not None:
                kw["cutoffs"] = r.cutoffs
            if r.stop is not None:
                kw["stop"] = r.stop
            eng.admit(j, r.input_ids, r.max_new, r.temperature, r.top_k, r.top_p, r.penalty, r.u, **kw, **feats)
            r.features, r.u = {}, None
            if long:
                self._prefilling = (j, r)
            else:
                self._register(r)       # one stream: a later admission's gather runs after this prefill's scatter
                self._started(j, r)

    def _register(self, r: _Request) -> None:
        """The request's prompt K / V are in its pages: its shareable pages join the prefix cache."""
        if r.prefix:
            self.pool.register(r.pages, r.prefix)

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
        state = torch.stack([eng.done, eng.cur_len] + ([eng.accepted] if self.lookup_k else [])).cpu()
        freed = 0
        for j in sorted(self._running):
            if not int(state[0, j]):
                continue
            r = self._running.pop(j)
            if self.lookup_k:
                self.accepted_drafts[r.rid] = int(state[2, j])
            if r.logprobs is not None:
                self.logprobs[r.rid] = eng.token_logprobs_of(j, int(state[1, j]) - int(r.input_ids.shape[1]), r.logprobs)
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
                tier = ""
                if self.pool.host_pages:
                    tier = f" and the host tier has {self.pool.host_free_pages} of {self.pool.host_pages} pages free"
                raise RuntimeError(f"request {head.rid} needs {need} KV pages but only {self.pool.free_pages} of "
                                   f"{self.pool.n_pages} are free: open sessions hold {self.pool.session_pages()}{tier}; close some")
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
                self._register(r)
                self._started(j, r)
        return results

    def pending(self) -> List[int]:
        pf = [] if self._prefilling is None else [self._prefilling[1].rid]
        return [r.rid for r in self._queue] + pf + [r.rid for r in self._running.values()]
