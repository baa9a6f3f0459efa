"""Prefix cache on the paged KV pool (serving.PagePool's reference counts and prefix index, and the scheduler's admission with
prefix_cache=True) on the host, with a stand-in engine, so no GPU is needed: which pages two prompts share, the caps on a hit,
the pool's invariants under a random sequence of operations, LRU eviction with descendants, all-or-nothing reservation,
first registration wins, and the argument check."""
import random

import pytest
import torch

from ultravox_b200 import serving
from ultravox_b200.serving import PAGE, PagePool


def check(pool: PagePool, holders=None):
    """The pool's invariants; ``holders`` (lists of pages held) gives the expected reference counts."""
    free, recl = set(pool._free), set(pool._reclaimable)
    held = {p for p in range(pool.n_pages) if pool._refs[p] > 0}
    assert len(free) == len(pool._free) and all(r >= 0 for r in pool._refs)
    assert not free & recl and not free & held and not recl & held
    assert free | recl | held == set(range(pool.n_pages))
    assert all(pool._refs[p] == 0 for p in free | recl)
    assert recl <= set(pool._key) and not free & set(pool._key)             # an indexed page is never free
    assert {p: k for k, p in pool._index.items()} == pool._key
    for p, (parent, toks) in pool._key.items():
        assert len(toks) == PAGE
        if parent is not None:
            assert parent in pool._key and p in pool._children[parent]
            assert pool._refs[p] == 0 or pool._refs[parent] > 0             # a held child has a held parent
    assert all(c in pool._key and pool._key[c][0] == p for p, cs in pool._children.items() for c in cs)
    if holders is not None:
        want = [0] * pool.n_pages
        for pages in holders:
            for p in pages:
                want[p] += 1
        assert want == pool._refs
    assert pool.free_pages == len(free) + len(recl) and pool.cached_pages == len(pool._key)


def toks(seed, n_pages, vary=None):
    """n_pages pages of token ids; ``vary`` = (page, offset): that one id differs."""
    rng = random.Random(seed)
    ids = [rng.randrange(1000) for _ in range(n_pages * PAGE)]
    if vary is not None:
        ids[vary[0] * PAGE + vary[1]] += 1000
    return tuple(tuple(ids[i:i + PAGE]) for i in range(0, len(ids), PAGE))


def donor(pool, pt, positions=None):
    pages = pool.reserve(positions or len(pt) * PAGE + 10)
    pool.register(pages, pt)
    return pages


# ------------------------------------------------------------------------------------------------ PagePool
@pytest.mark.parametrize("i", [0, 1, 3, 4])
def test_prompts_differing_in_page_i_share_pages_before_it(i):
    pool = PagePool(16)
    a = toks(0, 5)
    pa = donor(pool, a)
    b = toks(0, 5, vary=(i, 17))
    assert b[:i] == a[:i] and b[i] != a[i]
    assert pool.match(b) == pa[:i]
    pb = pool.reserve(5 * PAGE + 10, shared=pool.match(b))
    assert pb[:i] == pa[:i] and not set(pb[i:]) & set(pa)
    pool.register(pb, b)
    assert pool.cached_pages == 5 + (5 - i)       # b's own chain continues from the shared page i - 1
    assert pool.match(b) == pb[:5] and pool.match(a) == pa[:5]
    check(pool, [pa, pb])
    pool.release(pb)
    pool.release(pa)
    check(pool, [])
    assert pool.free_pages == 16


def test_duplicate_registration_keeps_the_first_page():
    pool = PagePool(16)
    t = toks(1, 3)
    pa = pool.reserve(3 * PAGE + 5)                 # two requests admitted before either registered
    pb = pool.reserve(3 * PAGE + 5)
    pool.register(pa, t)
    pool.register(pb, t)
    assert pool.match(t) == pa[:3] and pool.cached_pages == 3
    check(pool, [pa, pb])
    pool.release(pb)                                # the newcomer's pages were private: back to the free list
    assert len(pool._free) == 16 - 4 and len(pool._reclaimable) == 0
    pool.release(pa)
    assert len(pool._reclaimable) == 3 and pool.free_pages == 16
    check(pool, [])


def test_eviction_is_lru_and_takes_descendants():
    pool = PagePool(8)
    a = donor(pool, toks(2, 3), 3 * PAGE)           # chain a0 - a1 - a2
    b = donor(pool, toks(3, 2), 2 * PAGE)           # chain b0 - b1
    pool.release(a)                                 # a's pages released before b's: a is older
    pool.release(b)
    assert pool.free_pages == 8 and len(pool._free) == 3 and pool.cached_pages == 5
    order = list(pool._reclaimable)
    assert order == [a[2], a[1], a[0], b[1], b[0]]  # a chain's tail is released before its head
    new = pool.reserve(4 * PAGE)                    # 3 free pages, then evict the oldest (a's tail)
    assert a[2] in new and pool.match(toks(2, 3)) == a[:2] and pool.match(toks(3, 2)) == b and pool.evicted == 1
    check(pool, [new])
    pool.release(new)
    # a child is always released before its parent, so LRU takes leaves first; with a chain's first page made the oldest by
    # hand, evicting it unindexes the pages below it too (they could no longer be reached) and frees them
    pool = PagePool(6)
    a = donor(pool, toks(4, 3), 3 * PAGE)
    b = donor(pool, toks(5, 1), PAGE)
    pool.release(a)
    pool.release(b)
    pool._reclaimable.move_to_end(a[0], last=False)
    got = pool.reserve(3 * PAGE)                    # 2 free + one eviction of a0, which frees a1 and a2 as well
    assert pool.match(toks(4, 3)) == [] and pool.match(toks(5, 1)) == b
    assert pool.cached_pages == 1 and len(pool._free) == 2 and pool.evicted == 3
    check(pool, [got])


def test_waiting_request_holds_nothing():
    pool = PagePool(4)
    t = toks(6, 2)
    pa = donor(pool, t, 2 * PAGE)
    pool.release(pa)                                # both cached pages reclaimable
    other = pool.reserve(2 * PAGE)                  # takes the 2 free pages
    before = (list(pool._free), list(pool._reclaimable), list(pool._refs))
    assert pool.reserve(5 * PAGE, shared=pool.match(t)) is None     # needs 3 new pages besides the 2 shared: only 0 left
    assert (list(pool._free), list(pool._reclaimable), list(pool._refs)) == before
    got = pool.reserve(2 * PAGE + 1, shared=pool.match(t))          # shared pages are not counted as evictable for itself
    assert got is None
    pool.release(other)
    got = pool.reserve(4 * PAGE, shared=pool.match(t))
    assert got[:2] == pa and pool.free_pages == 0
    check(pool, [got])


def test_session_shares_then_keeps_its_references():
    pool = PagePool(12)
    t = toks(7, 2)
    pa = donor(pool, t, 3 * PAGE)
    sid = pool.open_session()
    p1 = pool.reserve(3 * PAGE, sid, shared=pool.match(t))
    assert p1[:2] == pa[:2]
    pool.release(pa)
    pool.release(p1, sid, kv_len=2 * PAGE + 30)     # the session keeps the shared pages and its own third page
    assert pool.session(sid).pages == p1[:3] and pool._refs[pa[0]] == 1
    with pytest.raises(ValueError, match="first turn"):
        pool.reserve(4 * PAGE, sid, shared=pool.match(t))
    p2 = pool.reserve(4 * PAGE, sid)
    assert p2[:3] == p1[:3]
    pool.release(p2, sid, kv_len=4 * PAGE - 1)
    check(pool, [pool.session(sid).pages])
    pool.close_session(sid)
    check(pool, [])
    assert pool.free_pages == 12 and pool.cached_pages == 2


def test_random_operations_keep_invariants():
    rng = random.Random(1234)
    pool = PagePool(24)
    prompts = [toks(100 + k, 4) for k in range(3)] + [toks(100, 4, vary=(2, 5)), toks(101, 4, vary=(1, 0))]
    running, sessions = [], {}                      # running: (pages, sid or None, prefix)
    for step in range(3000):
        op = rng.choice(["admit", "admit", "register", "retire", "open", "close"])
        if op == "open" and len(sessions) < 4:
            sessions[pool.open_session()] = False
        elif op == "close" and sessions:
            sid = rng.choice([s for s, busy in sessions.items() if not busy] or [None])
            if sid is not None:
                pool.close_session(sid)
                del sessions[sid]
        elif op == "admit":
            pt = rng.choice(prompts)[:rng.randint(0, 4)]
            positions = len(pt) * PAGE + rng.randint(1, 150)
            idle = [s for s, busy in sessions.items() if not busy]
            sid = rng.choice(idle + [None, None])
            if sid is not None and pool.session(sid).kv_len:
                shared, pt = [], ()
            else:
                shared = pool.match(pt[:(positions - 1) // PAGE])
            pages = pool.reserve(positions, sid, shared)
            if pages is None:
                check(pool)
                continue
            assert pages[:len(shared)] == shared
            running.append([pages, sid, pt, False])
            if sid is not None:
                sessions[sid] = True
                pool.session(sid).busy = True
        elif op == "register" and running:
            r = rng.choice(running)
            if not r[3]:
                pool.register(r[0], r[2])
                r[3] = True
        elif op == "retire" and running:
            pages, sid, _, _ = running.pop(rng.randrange(len(running)))
            if sid is None:
                pool.release(pages)
            else:
                pool.release(pages, sid, rng.randint(len(pages) * PAGE - 63, len(pages) * PAGE) - 1)
                sessions[sid] = False
        holders = [r[0] for r in running if r[1] is None] + [pool.session(s).pages for s in sessions]
        check(pool, holders)
    for pages, sid, _, _ in running:
        pool.release(pages, sid, 0) if sid is not None else pool.release(pages)
    for sid in list(sessions):
        pool.close_session(sid)
    check(pool, [])
    assert pool.free_pages == 24


# ------------------------------------------------------------------------------------------------ the scheduler
class _StubEngine:
    def __init__(self, model, slots, max_len, kv_pages=None, eos_token_ids=None, pad_token_id=0, use_graph=True):
        self.slots, self.max_len = slots, max_len
        self.busy = [False] * slots
        self.pos = torch.zeros(slots, dtype=torch.int32)
        self.prefilling = None
        self.admitted = []

    def admit(self, slot, input_ids, max_new, *args, past=0, pages=None, **features):
        self.busy[slot] = True
        S = int(input_ids.shape[1])
        if S - past > serving.PREFILL_ROWS:
            self.prefilling = slot
        self.admitted.append((slot, S, past, list(pages)))


def _sched(monkeypatch, slots=4, max_len=2048, kv_pages=64):
    monkeypatch.setattr(serving, "PagedSlotDecodeEngine", _StubEngine)
    sched = serving.SlotScheduler(None, slots=slots, max_len=max_len, kv_pages=kv_pages, prefix_cache=True)
    monkeypatch.setattr(sched, "_started", lambda j, r: sched._running.__setitem__(j, r))
    return sched


def request(sys_ids, n_user, seed, audio_at=None, n_audio=20):
    g = torch.Generator().manual_seed(seed)
    ids = torch.cat([torch.tensor(sys_ids, dtype=torch.int64), torch.randint(0, 1000, (n_user,), generator=g)])[None]
    feats = dict(input_ids=ids)
    if audio_at is not None:
        feats["audio_token_start_idx"] = torch.tensor([audio_at, audio_at + n_audio + 3])
    return feats


def _retire_all(sched):
    for j, r in list(sched._running.items()):
        sched.pool.release(r.pages, r.session, int(r.input_ids.shape[1]))
        sched.engine.busy[j] = False
    sched._running.clear()


def test_prefix_cache_needs_kv_pages():
    with pytest.raises(ValueError, match="kv_pages"):
        serving.SlotScheduler(None, slots=2, max_len=64, prefix_cache=True)


def test_hit_caps(monkeypatch):
    """The hit is capped at the first audio row, at S - 1 and to whole pages."""
    sched = _sched(monkeypatch)
    sys_ids = list(range(1, 1 + 3 * PAGE))
    a = sched.submit(request(sys_ids, 30, 0), max_new_tokens=4)              # no audio: registers 3 full pages
    sched._admit()
    assert sched.cached_tokens[a] == 0 and sched.cached_pages == 3
    cases = [(request(sys_ids, 30, 1), 3 * PAGE),                          # every shared page
             (request(sys_ids, 30, 2, audio_at=2 * PAGE + 10), 2 * PAGE),  # first audio row inside page 2
             (request(sys_ids, 30, 3, audio_at=2 * PAGE), 2 * PAGE),       # first audio row at a page boundary
             (request(sys_ids, 30, 4, audio_at=0), 0),
             (request(sys_ids, 0, 5), 2 * PAGE),                # S = 192: at most S - 1 rows, so 2 pages
             (request(sys_ids, 1, 6), 3 * PAGE),                      # S = 193: S - 1 = 192 = 3 whole pages
             (request(sys_ids[:PAGE + 40], 0, 7), PAGE)]                   # a partial page is recomputed
    for feats, want in cases:
        rid = sched.submit(feats, max_new_tokens=4)
        sched._admit()
        slot, S, past, pages = sched.engine.admitted[-1]
        assert sched.cached_tokens[rid] == past == want, (S, want)
        assert pages[:want // PAGE] == sched.engine.admitted[0][3][:want // PAGE]
        _retire_all(sched)
    assert sched.free_pages == 64


def _last_chunk(sched):
    """What run() does once the engine has run the prefilling request's last chunk."""
    sched.engine.prefilling = None
    j, r = sched._prefilling
    sched._prefilling = None
    sched._register(r)
    sched._started(j, r)
    return r


def test_chunked_donor_registers_after_its_last_chunk(monkeypatch):
    sched = _sched(monkeypatch)
    sys_ids = list(range(1, 1 + 3 * PAGE))
    a = sched.submit(request(sys_ids, 100, 0), max_new_tokens=4)             # 292 rows: chunked
    b = sched.submit(request(sys_ids, 20, 1), max_new_tokens=4)              # queued behind it, B = 1
    sched._admit()
    assert sched._prefilling[1].rid == a
    assert sched.cached_tokens == {a: 0, b: 0}                               # no hit on pages still being written
    pa, pb = sched._prefilling[1].pages, sched._running[1].pages
    assert sched.pool.match(sched._running[1].prefix) == pb[:3]              # b's own pages, registered at its admission
    _last_chunk(sched)
    assert sched.pool.match(sched._running[0].prefix) == pb[:3] and sched.cached_pages == 3     # the first registration won
    c = sched.submit(request(sys_ids, 20, 2), max_new_tokens=4)
    sched._admit()
    assert sched.cached_tokens[c] == 3 * PAGE and sched.engine.admitted[-1][3][:3] == pb[:3]
    _retire_all(sched)
    # a chunked donor alone: nothing is cached until its last chunk, then a request hits its pages; a hit whose suffix is
    # still over 256 rows is prefilled in chunks from P
    other = list(range(500, 500 + 3 * PAGE))
    d = sched.submit(request(other, 100, 3), max_new_tokens=4)
    sched._admit()
    assert sched.cached_pages == 3 and sched.pool.match(toks_of(other)) == []
    pd = _last_chunk(sched).pages
    assert sched.pool.match(toks_of(other)) == pd[:3]
    e = sched.submit(request(other, 20, 4), max_new_tokens=4)
    f = sched.submit(request(other, 300, 5), max_new_tokens=4)
    sched._admit()
    assert sched.cached_tokens[e] == sched.cached_tokens[f] == 3 * PAGE
    assert sched._prefilling[1].rid == f and sched.engine.admitted[-1][1:3] == (3 * PAGE + 300, 3 * PAGE)
    assert sched.engine.admitted[-1][3][:3] == pd[:3]


def toks_of(ids):
    return tuple(tuple(ids[i:i + PAGE]) for i in range(0, len(ids) // PAGE * PAGE, PAGE))


def test_session_first_turn_hits_later_turns_do_not(monkeypatch):
    sched = _sched(monkeypatch)
    sys_ids = list(range(1, 1 + 2 * PAGE))
    sched.submit(request(sys_ids, 10, 0), max_new_tokens=4)
    sched._admit()
    sid = sched.open_session()
    t1 = sched.submit(request(sys_ids, 10, 1), max_new_tokens=4, session=sid)
    sched._admit()
    assert sched.cached_tokens[t1] == 2 * PAGE
    shared = sched.engine.admitted[0][3][:2]
    assert sched.pool.session(sid).pages[:2] == shared
    _retire_all(sched)
    assert sched.pool.session(sid).pages[:2] == shared and sched.pool._refs[shared[0]] == 1
    prev = sched.pool.session(sid).kv_len
    t2 = sched.submit(request(sys_ids + [5] * (prev - len(sys_ids)), 30, 2), max_new_tokens=4, session=sid)
    sched._admit()
    assert sched.cached_tokens[t2] == 0 and sched.engine.admitted[-1][2] == prev
    _retire_all(sched)
    sched.close_session(sid)
    assert sched.free_pages == 64


def test_run_error_counts_reclaimable_pages(monkeypatch):
    sched = _sched(monkeypatch, kv_pages=6)
    sid = sched.open_session()
    sched.pool.release(sched.pool.reserve(4 * PAGE, sid), sid, kv_len=4 * PAGE)     # a session keeps 4 pages
    p = sched.pool.reserve(2 * PAGE)
    sched.pool.register(p, toks(9, 2))
    sched.pool.release(p)                                                            # 2 reclaimable cached pages
    assert sched.free_pages == 2 and sched.cached_pages == 2
    sched.submit(request(list(range(1, 200)), 0, 0), max_new_tokens=100)           # 5 pages
    with pytest.raises(RuntimeError, match="only 2 of 6 are free: open sessions hold 4"):
        sched.run()
