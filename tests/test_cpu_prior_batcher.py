"""CPU: the prior batcher (kandinsky2/batching.py, PriorBatcher) and the decoder batcher fed by it -- the per-slot UnCLIP
tables, a request's draws against image_emb / emb2emb, every refusal with nothing queued, the order in which decoder requests
waiting on prior requests join the decoder queue, and how many prior and decoder replays one step() issues."""
import collections
import types

import numpy as np
import pytest
import torch

from kandinsky2.batching import Batcher, PriorBatcher, SlotSteps, _PriorRequest, _Request, _SlotBatcher, prior_request_tables
from kandinsky2.model.prior import PriorEmbedder22, UnCLIPSchedule

D = 8


@pytest.mark.parametrize("steps", [2, 10, 25, 1000])
def test_prior_tables_are_the_unclip_schedule(steps):
    """Every kept row, full and truncated: the timesteps and k2_sampler_step rows of UnCLIPSchedule, rounded once to fp32, and
    a truncated table is the full table's tail."""
    full_ts, full_coef = prior_request_tables(steps)
    for keep in sorted({None, 1, steps // 2 or 1, steps - 1 or 1, steps}, key=lambda k: -1 if k is None else k):
        ts, coef = prior_request_tables(steps, keep)
        sched = UnCLIPSchedule(steps, keep=keep)
        n = steps if keep is None else keep
        assert ts.dtype == coef.dtype == torch.float32 and ts.shape == (n,) and coef.shape == (n, 8)
        assert np.array_equal(ts.numpy(), sched.timesteps.astype(np.float32))
        assert np.array_equal(coef.numpy(), sched.rows().astype(np.float32))
        assert torch.equal(ts, full_ts[steps - n:]) and torch.equal(coef, full_coef[steps - n:])
    assert full_ts[0].item() == 999.0 and full_ts[-1].item() == 0.0
    assert full_coef[-1, 6].item() == 0.0 and bool((full_coef[:-1, 6] == 1.0).all())   # no noise at t = 0 only


def _clip_text(prompts):
    outs = []
    for p in prompts:
        g = torch.Generator().manual_seed(len(p) + 17 * sum(map(ord, p)))
        outs.append((torch.randn(D, generator=g), torch.randn(3, D, generator=g), torch.arange(3) < 1 + len(p) % 2))
    return tuple(torch.stack(t) for t in zip(*outs))


def _bare_prior(slots=2):
    """A PriorBatcher without a GPU: a real PriorEmbedder22 on the CPU around a stand-in prior, its slots on the CPU, no plan
    and no graph."""
    calls = []

    def clip_text(prompts):
        calls.append(list(prompts))
        return _clip_text(prompts)
    emb = PriorEmbedder22(types.SimpleNamespace(clip_dim=D, _packed="w", _lora=None), clip_text, torch.zeros(D), torch.ones(D),
                          clip_image=lambda img: torch.linspace(-1, 1, D)[None], prior_steps=10, seed=3)
    pb = object.__new__(PriorBatcher)
    pb.embedder, pb._weights0 = emb, ("w", None)
    _SlotBatcher.__init__(pb, slots)
    pb.slots = SlotSteps(slots, (4, 1, D // 4), PriorBatcher.MAX_STEPS, "cpu")
    return pb, calls


@pytest.mark.parametrize("guidance", [4.0, 1.0])
def test_a_request_draws_what_image_emb_and_emb2emb_draw(guidance):
    pb, _ = _bare_prior()
    emb = pb.embedder
    r = pb.request("a red cat", prior_steps=7, prior_guidance_scale=guidance, negative_prior_prompt="ugly")
    steps, g, rows, gen = emb._call_args("a red cat", 1, 7, guidance, "ugly")
    x_T = torch.randn(1, D, generator=gen)
    noise = torch.randn(7, 1, D, generator=gen)
    assert r.steps == 7 and r.guidance == g == guidance and torch.equal(r.x, x_T) and torch.equal(r.noise, noise)
    assert all(torch.equal(a, b) for a, b in zip(r.rows, rows))
    ts, coef = prior_request_tables(7)
    assert torch.equal(r.ts, ts) and torch.equal(r.coef, coef)
    image = torch.randn(D)
    r2 = pb.request("a red cat", prior_steps=7, prior_guidance_scale=guidance, image=image, strength=0.6)
    keep = 4   # int(7 * 0.6)
    *_, gen = emb._call_args("a red cat", 1, 7, guidance, None)
    z = torch.randn(1, D, generator=gen)
    noise = torch.randn(keep, 1, D, generator=gen)
    sched = UnCLIPSchedule(7, keep=keep)
    assert r2.steps == keep and torch.equal(r2.noise, noise) and torch.equal(r2.x, sched.start_latent(image[None], z))
    assert torch.equal(r2.ts, prior_request_tables(7, keep)[0])
    r3 = pb.request("a red cat", image=image)   # emb2emb's default strength (0.3) and the embedder's 10 steps
    assert r3.steps == 3 and not pb.queue.waiting and not pb._requests


@pytest.mark.parametrize("kw, match", [
    (dict(prior_steps=1), "prior_steps"),
    (dict(prior_steps=1001), "prior_steps"),
    (dict(prior_steps=2.0), "prior_steps"),
    (dict(prior_steps=True), "prior_steps"),
    (dict(strength=0.5), "strength without image"),
    (dict(image=torch.zeros(D), strength=-0.1), "strength"),
    (dict(image=torch.zeros(D), strength=1.5), "strength"),
    (dict(image=torch.zeros(D), strength="0.5"), "strength"),
    (dict(image=torch.zeros(D), strength=0.05), "keeps no step"),
    (dict(image=torch.zeros(2, D)), "image"),
    (dict(image=torch.zeros(D + 1)), "image"),
    (dict(image=torch.zeros(1, D - 1)), "image"),
    (dict(image=torch.zeros(1, 1, D)), "image"),
])
def test_prior_submit_refusals_queue_nothing(kw, match):
    pb, calls = _bare_prior()
    with pytest.raises(ValueError, match=match):
        pb.submit("a red cat", **kw)
    assert not pb.queue.waiting and not pb._requests and pb._next_handle == 0 and not calls


def test_prior_batcher_refuses_a_bad_max_batch():
    for bad in (0, -1, 1.0, True, None):
        with pytest.raises(ValueError, match="max_batch"):
            PriorBatcher(None, bad)


def test_decoder_batcher_refuses_prior_slots_without_a_prior_batcher():
    from kandinsky2.pipelines import Kandinsky2_1, Kandinsky2_2, SyntheticEmbedder
    pipe = object.__new__(Kandinsky2_2)
    pipe.task_type, pipe.embedder = "text2img", SyntheticEmbedder(D)
    for bad in (-1, 1.5, True, "2"):
        with pytest.raises(ValueError, match="prior_slots"):
            Batcher(pipe, 2, 64, 64, prior_slots=bad)
    with pytest.raises(ValueError, match="prior_slots"):
        Batcher(pipe, 2, 64, 64, prior_slots=2)
    import inspect
    assert "prior_slots" in inspect.signature(Kandinsky2_2.batcher).parameters
    assert "prior_slots" not in inspect.signature(Kandinsky2_1.batcher).parameters


# ------------------------------------------------------------------------------------------------------------------------------
# the decoder batcher fed by prior requests, on bare objects
# ------------------------------------------------------------------------------------------------------------------------------
class _ScriptedPrior:
    """Stands in for a PriorBatcher: enqueue hands out handles, step() finishes the prior handles the script names."""

    def __init__(self, script):
        self.script, self.n = list(script), 0

    def enqueue(self, r):
        self.n += 1
        return self.n - 1

    def pending(self):
        return bool(self.script)

    def step(self):
        return {h: torch.full((1, D), float(h)) for h in self.script.pop(0)}


def _bare_batcher(prior, slots=2):
    b = object.__new__(Batcher)
    b.max_steps, b.prior, b._held, b._waiting_on = 50, prior, {}, {}
    _SlotBatcher.__init__(b, slots)
    return b


def _request(steps, positive, negative):
    r = _Request()
    r.ts, r.positive, r.negative, r.lora = torch.zeros(steps), positive, negative, None
    return r


def _prior_request(steps=3):
    r = _PriorRequest()
    r.steps = steps
    return r


def test_requests_waiting_on_prior_handles_join_the_decoder_queue_in_order():
    """Prior handles 0 / 1 are request 0's positive / negative, 2 / 3 request 1's, 4 request 3's positive, 5 / 6 request 4's;
    request 2 brings its embeddings and joins at once.  Each joins when its last embedding is done, and requests that become
    ready at the same prior step join in submit order, whatever order their prior requests finished in."""
    prior = _ScriptedPrior([[3, 2], [0], [6, 4], [5, 1]])
    b = _bare_batcher(prior)
    zero = torch.zeros(1, D)
    hs = [b._enqueue(_request(4, _prior_request(), _prior_request())),
          b._enqueue(_request(5, _prior_request(), _prior_request())),
          b._enqueue(_request(6, zero, zero)),
          b._enqueue(_request(7, _prior_request(), zero)),
          b._enqueue(_request(8, _prior_request(), _prior_request()))]
    assert hs == [0, 1, 2, 3, 4]
    assert b._waiting_on == {0: (0, "positive"), 1: (0, "negative"), 2: (1, "positive"), 3: (1, "negative"), 4: (3, "positive"),
                             5: (4, "positive"), 6: (4, "negative")}
    assert [h for h, _ in b.queue.waiting] == [2] and b._held == {0: 2, 1: 2, 3: 1, 4: 2}
    order = []
    for _ in range(4):
        assert b._prior_step()
        order.append([h for h, _ in b.queue.waiting])
    assert order == [[2, 1], [2, 1], [2, 1, 3], [2, 1, 3, 0, 4]]
    assert not b._held and not b._waiting_on
    r0, r1, r4 = b._requests[0], b._requests[1], b._requests[4]
    assert (r0.positive[0, 0].item(), r0.negative[0, 0].item(), r1.positive[0, 0].item(), r1.negative[0, 0].item()) == (0, 1, 2, 3)
    assert r4.positive[0, 0].item() == 5 and r4.negative[0, 0].item() == 6 and b._requests[3].negative is zero
    assert [s for _, s in b.queue.waiting] == [6, 5, 7, 4, 8]


# ------------------------------------------------------------------------------------------------------------------------------
# the scheduling rule: replays per step(), with both graphs replaced by counters
# ------------------------------------------------------------------------------------------------------------------------------
class _Counter:
    def __init__(self):
        self.n = 0

    def replay(self):
        self.n += 1


class _Event:
    def record(self):
        pass

    def synchronize(self):
        pass


def _scheduled(monkeypatch, slots=2, prior_slots=2):
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    pb, _ = _bare_prior(prior_slots)
    pb.graph = _Counter()
    pb._stage = lambda s, r: None
    b = _bare_batcher(pb, slots)
    b.graph, b._events, b.w_map, b.h, b.w = _Counter(), collections.deque(), None, 64, 64
    b.slots = SlotSteps(slots, (4, 1, 1), b.max_steps, "cpu")
    b._weights0 = ("unet",)
    b.pipe = types.SimpleNamespace(model=types.SimpleNamespace(_packed="unet"), _finish=lambda x, h, w: ["image"])
    b._stage = lambda s, r: None
    return b, pb


def _prompt(b, decoder_steps, *prior_steps):
    """A decoder request whose positive (and negative, given two counts) embeddings are prior requests of those steps."""
    reqs = [_prior_request(k) for k in prior_steps] + [torch.zeros(1, D)] * (2 - len(prior_steps))
    return b._enqueue(_request(decoder_steps, *reqs))


def _replays(b, pb):
    before = (pb.graph.n, b.graph.n)
    b.step()
    return pb.graph.n - before[0], b.graph.n - before[1]


def test_a_free_decoder_slot_with_nothing_ready_runs_the_prior_back_to_back(monkeypatch):
    """Burst: the first step() replays the prior until its first request finishes (the fewest steps of the busy prior
    slots), then the decoder step; the next step() does it again for the other slot."""
    b, pb = _scheduled(monkeypatch)
    a = _prompt(b, 10, 3)
    c = _prompt(b, 10, 6)
    assert _replays(b, pb) == (3, 1) and b.queue.holder == [a, None]
    assert _replays(b, pb) == (3, 1) and b.queue.holder == [a, c]
    assert _replays(b, pb) == (0, 1)
    # a request waiting on two prior requests: the burst stops at the first of them, and the decoder slot stays free
    b2, pb2 = _scheduled(monkeypatch)
    d = _prompt(b2, 2, 4, 2)
    assert _replays(b2, pb2) == (2, 0) and b2.queue.holder == [None, None] and b2._held == {d: 1}
    assert _replays(b2, pb2) == (2, 1) and b2.queue.holder == [d, None]


def test_busy_decoder_slots_take_one_prior_step_per_step(monkeypatch):
    """Trickle: with every decoder slot busy (or a ready request waiting for one), each step() replays one prior step, then
    the decoder step; once the prior batch is empty, only the decoder."""
    b, pb = _scheduled(monkeypatch, slots=1)
    z = torch.zeros(1, D)
    first = b._enqueue(_request(6, z, z))
    assert _replays(b, pb) == (0, 1) and b.queue.holder == [first]
    h = _prompt(b, 3, 3)
    assert [_replays(b, pb) for _ in range(3)] == [(1, 1)] * 3
    assert [hh for hh, _ in b.queue.waiting] == [h] and not b._held
    assert [_replays(b, pb) for _ in range(2)] == [(0, 1)] * 2
    assert b.queue.holder == [None]
    assert _replays(b, pb) == (0, 1) and b.queue.holder == [h]
    # a ready request waits while the decoder slot is busy: a new prompt then trickles instead of bursting
    h2 = _prompt(b, 2, 5)
    assert [_replays(b, pb) for _ in range(2)] == [(1, 1)] * 2
    out = b.run()   # the decoder slot frees up: the rest of h2's prior steps back to back
    assert list(out) == [h2] and pb.graph.n == 3 + 5 and not b._held and not pb.pending()


def test_emb2emb_image_embedding_keeps_its_flat_batch_form():
    """emb2emb still takes a flat [B * D] embedding at batch B (reshaped to [B, D]); a prior request takes [1, D] / [D] only."""
    pb, _ = _bare_prior()
    flat = torch.arange(2 * D, dtype=torch.float32)
    assert torch.equal(pb.embedder._image_embedding(flat, 2), flat.reshape(2, D))
    with pytest.raises(ValueError, match="image"):
        pb.request("a red cat", image=flat)


def test_a_failed_prior_admission_drops_its_decoder_request(monkeypatch):
    """When staging a prior request fails inside step(), the error propagates, the decoder request waiting on it is dropped
    with it (the result of its other prior request is discarded), and run() ends instead of waiting on it for ever."""
    b, pb = _scheduled(monkeypatch, slots=2, prior_slots=2)
    good = _prompt(b, 2, 2)
    bad = _prompt(b, 2, 3, 1)

    def stage(s, r):
        if r.steps == 1:
            raise RuntimeError("staging failed")
    pb._stage = stage
    with pytest.raises(RuntimeError, match="staging failed"):
        b.run()   # the second step() admits the third prior request
    assert bad not in b._requests and bad not in b._held and not b._waiting_on
    out = b.run()
    assert list(out) == [good] and not b._held
    while pb.pending():   # the dropped request's positive embedding finishes and is discarded
        assert not b._prior_step() or not b.queue.waiting
