"""Continuous batching against static batches on a serving workload.

64 independent requests to the 8B backbone with the large-v3 encoder (`preset("v0_5_8b")`, random weights), all submitted at
t = 0.  Each is one clip of 5, 10, 20 or 30 s between 8 and 5 text tokens, with a budget of 16-256 new tokens drawn uniformly
(fixed seed).  There are no EOS ids (random weights almost never emit one), so each budget sets its reply length.  Greedy.

Arms, alternated over `--rounds` rounds in one process after a warm-up of each:
- static: batches of 8 in submission order, left-padded as `LocalInference.infer_batch` collates them, one `generate()` per
  batch with `max_new_tokens` = the batch's largest budget (every row decodes until the longest reply ends);
- slots: `serving.SlotScheduler` with 8 slots (one engine, captured once before the rounds).

Per arm: wall time (host clock, synchronised), useful tokens per second (the sum of the budgets over the wall time), decode
milliseconds per step (CUDA events around every decode step), time to first token p50 / p90 over the 64 requests (CUDA events
from t = 0 to the request's first picked token) and the share of decode row-steps (rows x steps) that decode padding or idle slots.
The slots arm also reports the inter-token gaps of every request (p50 / p99 over all gaps, the largest gap of each request at
p50 and its maximum; from the same per-step events) and, apart, the mean time of plain steps and of mixed steps (steps that
carry a chunk of a long prompt, see below).

`--workload long`: the same 64 budgets, but each clip lasts 40-90 s, cut into 30 s encoder chunks as the processor does
(`processing.frame_chunks`), so prompts hold 264-577 rows.  Every such prompt is over the 256 rows up to which a prompt is
prefilled whole at admission, so the slot engine prefills it in chunks inside its decode steps; the default workload (at most
201 rows) never does.  `--arms slots` skips the static arm.

`--kv-pages N` adds the arm `paged` to the default / long workloads: the same scheduler on the paged KV cache
(`PagedSlotDecodeEngine`, N shareable 64-position pages), which must pick the same tokens at about the same step time.

`--workload conversations`: 32 conversations (`--requests`) x 4 turns (`--turns`); each turn is one 5 or 10 s clip between
8 and 5 text tokens with a budget of 16-256 new tokens, and the next turn of a conversation is submitted from the `on_tokens`
callback as soon as the previous reply arrives (its prompt: the conversation so far, then the new turn).  Arms:
- sessions: `SlotScheduler(kv_pages=N)` with one session per conversation, so each turn prefills only its new suffix;
- slots: the contiguous engine, each turn submitted as its whole conversation (prefilled again from position 0).
Per arm: wall time, tokens per second, TTFT p50 / p90 per turn index (from the turn's submission to its first token), plain
and mixed step times; the sessions arm also reports the admission gather + scatter of 4096 positions at these widths.

Prints the device name and power limit first, then one JSON line per arm."""
import argparse, json, os, statistics, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch
from sample_bench import device_info
from ultravox_b200 import ops

SR, PRE, POST = 16000, 8, 5


def make_requests(cfg, n, seed, workload="default"):
    from ultravox_b200.processing import frame_chunks
    rng = np.random.default_rng(seed)
    secs = rng.choice([5, 10, 20, 30] if workload == "default" else [40, 50, 60, 70, 80, 90], size=n)
    budgets = rng.integers(16, 257, size=n)
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for i in range(n):
        wave = torch.from_numpy(rng.standard_normal(int(secs[i]) * SR).astype(np.float32)).cuda()
        mel = ops.logmel(wave[None], cfg.audio_config.num_mel_bins)
        plan, _ = frame_chunks([mel.shape[-1]], 3000)          # one chunk per 30 s, continuations zero-padded to 3000 frames
        pieces = [torch.nn.functional.pad(mel[0, :, off:off + 3000], (0, 3000 - min(3000, mel.shape[-1] - off)) if cont else (0, 0))
                  for _, off, _, cont in plan]
        frames = [p[2] for p in plan]
        tok = [-(-f // 16) for f in frames]
        starts = [PRE + sum(tok[:k]) for k in range(len(tok))]
        ids = torch.randint(0, 128000, (1, PRE + sum(tok) + POST), generator=g)
        reqs.append(dict(feats=dict(input_ids=ids.cuda(), audio_values=torch.stack(pieces), audio_token_start_idx=torch.tensor(starts).cuda(),
                                    audio_lens=torch.tensor(frames).cuda(), audio_token_len=torch.tensor(tok, dtype=torch.int32).cuda(),
                                    audio_batch_size=torch.tensor([len(plan)]).cuda()),
                         budget=int(budgets[i])))
    return reqs


def make_conversations(cfg, n, turns, seed):
    """Per conversation, per turn: (new ids, clip features relative to them, budget)."""
    rng = np.random.default_rng(seed)
    g = torch.Generator().manual_seed(seed)
    convs = []
    for _ in range(n):
        conv = []
        for _ in range(turns):
            wave = torch.from_numpy(rng.standard_normal(int(rng.choice([5, 10])) * SR).astype(np.float32)).cuda()
            mel = ops.logmel(wave[None], cfg.audio_config.num_mel_bins)
            tok = -(-mel.shape[-1] // 16)
            ids = torch.randint(0, 128000, (1, PRE + tok + POST), generator=g).cuda()
            conv.append(dict(ids=ids, mel=mel, frames=mel.shape[-1], tok=tok, budget=int(rng.integers(16, 257))))
        convs.append(conv)
    return convs


def turn_features(prev, t):
    """The conversation so far (``prev`` ids, or nothing) followed by turn t's ids, with turn t's clip spliced after them."""
    P = 0 if prev is None else prev.shape[1]
    ids = t["ids"] if prev is None else torch.cat([prev, t["ids"]], dim=1)
    return dict(input_ids=ids, audio_values=t["mel"], audio_token_start_idx=torch.tensor([P + PRE]).cuda(),
                audio_lens=torch.tensor([t["frames"]]).cuda(), audio_token_len=torch.tensor([t["tok"]], dtype=torch.int32).cuda(),
                audio_batch_size=torch.tensor([1]).cuda())


def run_conversations(sched, convs, sessions):
    """Serves every conversation turn by turn; returns (wall, {turn: [ttft ms]}, step ms, (plain, mixed) step ms)."""
    eng = sched.engine
    marks, plain = [], eng.step

    def timed():
        mixed = getattr(eng, "prefilling", None) is not None
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        plain()
        b.record()
        marks.append((a, b, mixed))

    eng.step = timed
    state, submitted = {}, {}

    def submit(c, t, prev, sid):
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        rid = sched.submit(turn_features(prev, convs[c][t]), max_new_tokens=convs[c][t]["budget"], session=sid)
        state[rid], submitted[rid] = (c, t, sid), ev

    def on_tokens(rid, seq):
        c, t, sid = state[rid]
        if t + 1 < len(convs[c]):
            submit(c, t + 1, seq, sid)
        elif sid is not None:
            sched.close_session(sid)

    torch.cuda.synchronize()
    w0 = time.perf_counter()
    for c in range(len(convs)):
        submit(c, 0, None, sched.open_session() if sessions else None)
    sched.run(on_tokens)
    torch.cuda.synchronize()
    wall = time.perf_counter() - w0
    eng.step = plain
    ttft = {}
    for rid, (c, t, _) in state.items():
        ttft.setdefault(t, []).append(submitted[rid].elapsed_time(sched.first_token[rid]))
    step = [a.elapsed_time(b) for a, b, _ in marks]
    split = {m: [x for x, (_, _, k) in zip(step, marks) if k == m] for m in (False, True)}
    return wall, ttft, step, split


def pages_copy_ms(eng, n=4096, reps=5):
    """Admission gather + scatter of n positions (every layer, K and V) between the one-row scratch and the pool."""
    pages = torch.arange(-(-n // ops.PAGE), dtype=torch.int32, device="cuda") % eng.kv_pages
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ops.kv_pages_copy(eng.cache.k, eng.cache.v, eng.pool_k, eng.pool_v, pages, 0, n, to_pages=False)
    a.record()
    for _ in range(reps):
        ops.kv_pages_copy(eng.cache.k, eng.cache.v, eng.pool_k, eng.pool_v, pages, 0, n, to_pages=False)
        ops.kv_pages_copy(eng.cache.k, eng.cache.v, eng.pool_k, eng.pool_v, pages, 0, n, to_pages=True)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main_conversations(args, model, cfg):
    from ultravox_b200.serving import SlotScheduler
    arms = args.arms.split(",")
    convs = make_conversations(cfg, args.requests, args.turns, args.seed)
    max_len = sum(PRE + t["tok"] + POST + t["budget"] for t in max(convs, key=lambda c: sum(t["tok"] + t["budget"] for t in c))) + 64
    max_len = max(max_len, 4096 + 64)
    kv_pages = args.kv_pages or 8 * (-(-max_len // ops.PAGE))
    scheds = {}
    if "sessions" in arms:
        scheds["sessions"] = (SlotScheduler(model, slots=8, max_len=max_len, kv_pages=kv_pages), True)
    if "slots" in arms:
        scheds["slots"] = (SlotScheduler(model, slots=8, max_len=max_len), False)
    warm = [c[:2] for c in convs[:8]]
    for sched, sess in scheds.values():
        run_conversations(sched, [[dict(t, budget=16) for t in c] for c in warm], sess)
    out = {a: [] for a in scheds}
    for _ in range(args.rounds):
        for a, (sched, sess) in scheds.items():
            out[a].append(run_conversations(sched, convs, sess))
    useful = sum(t["budget"] for c in convs for t in c)
    for arm, runs in out.items():
        walls = [r[0] for r in runs]
        k = walls.index(sorted(walls)[len(walls) // 2])
        wall, ttft, step, split = runs[k]
        line = {"bench": f"serve {len(convs)} conversations x {args.turns} turns, 8B + large-v3, clips 5-10 s, budgets 16-256, greedy",
                "arm": arm, "wall_s_median": wall, "wall_s_all": [round(w, 3) for w in walls], "useful_tokens": useful,
                "tokens_per_s": useful / wall, "max_len": max_len,
                "ttft_ms_p50_by_turn": [round(pct(ttft[t], 50), 2) for t in sorted(ttft)],
                "ttft_ms_p90_by_turn": [round(pct(ttft[t], 90), 2) for t in sorted(ttft)],
                "plain_step_ms_mean": statistics.fmean(split[False]) if split[False] else None, "plain_steps": len(split[False]),
                "mixed_step_ms_mean": statistics.fmean(split[True]) if split[True] else None, "mixed_steps": len(split[True])}
        if arm == "sessions":
            line["kv_pages"] = kv_pages
            line["gather_plus_scatter_4096_positions_ms"] = pages_copy_ms(scheds[arm][0].engine)
        print(json.dumps(line), flush=True)


def collate(batch):
    """Left padding, as the inference collator does: ids padded with 0 on the left, the audio start shifted, mel padded."""
    S = max(r["feats"]["input_ids"].shape[1] for r in batch)
    T = max(r["feats"]["audio_values"].shape[-1] for r in batch)
    ids, am, start, mels = [], [], [], []
    for r in batch:
        f = r["feats"]
        p = S - f["input_ids"].shape[1]
        ids.append(torch.nn.functional.pad(f["input_ids"], (p, 0)))
        am.append(torch.nn.functional.pad(torch.ones_like(f["input_ids"]), (p, 0)))
        start.append(f["audio_token_start_idx"] + p)
        mels.append(torch.nn.functional.pad(f["audio_values"], (0, T - f["audio_values"].shape[-1])))
    cat = lambda k: torch.cat([r["feats"][k] for r in batch])
    return dict(input_ids=torch.cat(ids), attention_mask=torch.cat(am), audio_token_start_idx=torch.cat(start),
                audio_values=torch.cat(mels), audio_lens=cat("audio_lens"), audio_token_len=cat("audio_token_len"),
                audio_batch_size=cat("audio_batch_size"))


class _Events:
    """A streamer that records a CUDA event per new token and never synchronises."""

    def __init__(self):
        self.events, self.seen_prompt = [], False

    def put(self, _):
        if not self.seen_prompt:
            self.seen_prompt = True
            return
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.events.append(e)

    def end(self):
        pass


def run_static(model, reqs, batch=8):
    t0 = torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    w0 = time.perf_counter()
    t0.record()
    ttft, steps_ms, row_steps = [], [], 0
    for i in range(0, len(reqs), batch):
        chunk = reqs[i:i + batch]
        n = max(r["budget"] for r in chunk)
        st = _Events()
        model.generate(**collate(chunk), max_new_tokens=n, streamer=st)
        ttft.append((st.events[0], len(chunk)))
        steps_ms.append(st.events)
        row_steps += (n - 1) * len(chunk)                   # the first token comes from the prefill
    torch.cuda.synchronize()
    wall = time.perf_counter() - w0
    first = [t0.elapsed_time(e) for e, k in ttft for _ in range(k)]
    step = [a.elapsed_time(b) for evs in steps_ms for a, b in zip(evs, evs[1:])]
    return wall, first, step, row_steps


class _FirstTokens(dict):
    """``SlotScheduler.first_token`` that also notes the scheduler's step count when each request's first token is picked."""

    def __init__(self, sched):
        super().__init__()
        self.sched, self.at = sched, {}

    def __setitem__(self, rid, ev):
        self.at[rid] = self.sched.steps
        super().__setitem__(rid, ev)


def run_slots(sched, reqs):
    eng = sched.engine
    marks = []
    plain = eng.step
    sched.first_token = _FirstTokens(sched)

    def timed():
        mixed = getattr(eng, "prefilling", None) is not None
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        plain()
        b.record()
        marks.append((a, b, mixed))

    eng.step = timed
    t0 = torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    w0 = time.perf_counter()
    t0.record()
    steps0 = sched.steps
    ids = [sched.submit(r["feats"], max_new_tokens=r["budget"]) for r in reqs]
    sched.run()
    torch.cuda.synchronize()
    wall = time.perf_counter() - w0
    eng.step = plain
    first = [t0.elapsed_time(sched.first_token[i]) for i in ids]
    step = [a.elapsed_time(b) for a, b, _ in marks]
    ends = [t0.elapsed_time(b) for _, b, _ in marks]
    # a request whose first token came at step count k gets its next tokens from steps k + 1, k + 2, ... (no EOS ids)
    gaps = []
    for i, r, f in zip(ids, reqs, first):
        k = sched.first_token.at[i] - steps0
        times = [f] + ends[k:k + r["budget"] - 1]
        gaps.append([b - a for a, b in zip(times, times[1:])])
    split = {m: [t for t, (_, _, x) in zip(step, marks) if x == m] for m in (False, True)}
    return wall, first, step, (sched.steps - steps0) * eng.slots, gaps, split


def pct(xs, q):
    return float(np.percentile(np.asarray(xs), q))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--requests", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--workload", choices=["default", "long", "conversations"], default="default")
    ap.add_argument("--arms", default=None, help="default: static,slots (conversations: sessions,slots)")
    ap.add_argument("--turns", type=int, default=4)
    ap.add_argument("--kv-pages", type=int, default=None)
    args = ap.parse_args()
    if args.arms is None:
        args.arms = "sessions,slots" if args.workload == "conversations" else "static,slots"
    if args.workload == "conversations" and "--requests" not in sys.argv:
        args.requests = 32
    arms = args.arms.split(",")
    if args.kv_pages and args.workload != "conversations" and "paged" not in arms:
        arms.append("paged")
    print(json.dumps({"device": device_info()}), flush=True)
    from ultravox_b200.config import preset
    from ultravox_b200.model import UltravoxModel
    from ultravox_b200.serving import SlotScheduler
    torch.set_grad_enabled(False)
    cfg = preset("v0_5_8b")
    model = UltravoxModel(cfg, device="cuda").init_random_(seed=42)
    if args.workload == "conversations":
        return main_conversations(args, model, cfg)
    reqs = make_requests(cfg, args.requests, args.seed, args.workload)
    useful = sum(r["budget"] for r in reqs)
    useful_steps = useful - len(reqs)                         # tokens picked by decode steps (the first comes from the prefill)
    max_len = max(r["feats"]["input_ids"].shape[1] for r in reqs) + 256
    c0 = time.perf_counter()
    sched = SlotScheduler(model, slots=8, max_len=max_len)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - c0
    paged = SlotScheduler(model, slots=8, max_len=max_len, kv_pages=args.kv_pages) if "paged" in arms else None
    warm = [dict(r, budget=16) for r in reqs[:8]]
    if "static" in arms:
        run_static(model, warm)
    run_slots(sched, warm)
    if paged is not None:
        run_slots(paged, warm)
    out = {a: [] for a in ("static", "slots", "paged") if a in arms}
    for _ in range(args.rounds):
        if "static" in arms:
            out["static"].append(run_static(model, reqs))
        out["slots"].append(run_slots(sched, reqs))
        if paged is not None:
            out["paged"].append(run_slots(paged, reqs))
    clips = "5-30 s" if args.workload == "default" else "40-90 s"
    for arm, runs in out.items():
        walls = [r[0] for r in runs]
        k = walls.index(sorted(walls)[len(walls) // 2])
        wall, first, step, row_steps = runs[k][:4]
        line = {"bench": f"serve {len(reqs)} requests, 8B + large-v3, clips {clips}, budgets 16-256, greedy", "arm": arm,
                "wall_s_median": wall, "wall_s_all": [round(w, 3) for w in walls], "useful_tokens": useful,
                "tokens_per_s": useful / wall, "decode_ms_per_step_mean": statistics.fmean(step), "decode_steps": len(step),
                "ttft_ms_p50": pct(first, 50), "ttft_ms_p90": pct(first, 90), "row_steps": row_steps,
                "wasted_row_step_share": 1.0 - useful_steps / row_steps}
        if arm in ("slots", "paged"):
            gaps, split = runs[k][4:]
            flat, worst = [g for gs in gaps for g in gs], [max(gs) for gs in gaps if gs]
            line.update(gap_ms_p50=pct(flat, 50), gap_ms_p99=pct(flat, 99), max_gap_ms_p50=pct(worst, 50), max_gap_ms_max=max(worst),
                        plain_step_ms_mean=statistics.fmean(split[False]) if split[False] else None, plain_steps=len(split[False]),
                        mixed_step_ms_mean=statistics.fmean(split[True]) if split[True] else None, mixed_steps=len(split[True]))
            line["engine_build_s"] = build_s
            line["launches_per_step"] = (sched if arm == "slots" else paged).engine.launches_per_step
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
