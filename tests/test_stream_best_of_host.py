"""CPU checks of best-of-n requests in the continuous-batching stream: the validation of each pulled request
(_stream_draws), the coercion of BestOfRequest items (_as_request, used by the list and the iterator paths alike), and
the slot-release rule of a request's candidates (_Candidates) driven through the first-in first-out slot choice
(_take_slots) on a host model of the scheduler."""
import pytest
import torch

from valle_b200.engine import BestOfRequest, StreamRequest, _as_request, _Candidates, _stream_draws, _take_slots


def _req(**kw):
    g = torch.Generator().manual_seed(0)
    r = StreamRequest(torch.randint(3, 100, (6,), generator=g), torch.randint(0, 1024, (9, 8), generator=g))
    return r._replace(**kw)


def test_best_of_draws_seed_s_plus_j():
    r, draws = _stream_draws(0, BestOfRequest(_req(seed=40, top_k=7, temperature=0.8, top_p=0.9, ras=(8, 0.25)), 3),
                             8, 4, False)
    assert r.num_beams == 1 and len(draws) == 3
    assert [d.seed for d in draws] == [40, 41, 42]
    assert all(d.top_k == 7 and d.temperature == 0.8 and d.top_p == 0.9 and d.ras_window == 8 for d in draws)
    # n == 1 is the plain request
    assert _stream_draws(0, BestOfRequest(_req(seed=40, top_k=7), 1), 8, 4, False)[1] == \
        _stream_draws(0, _req(seed=40, top_k=7), 8, 4, False)[1]
    # an unseeded greedy request draws with seed 0 (nothing is drawn)
    assert [d.seed for d in _stream_draws(0, _req(), 8, 4, False)[1]] == [0]


@pytest.mark.parametrize("item,what", [
    (BestOfRequest(_req(seed=1), 0), "request 3: num_samples must be an int >= 1"),
    (BestOfRequest(_req(seed=1), 2.0), "request 3: num_samples must be an int >= 1"),
    (BestOfRequest(_req(seed=1), True), "request 3: num_samples must be an int >= 1"),
    (BestOfRequest(_req(seed=1), 5), "request 3: num_samples=5 needs more than the 4 slots"),
    (BestOfRequest(_req(), 2), "request 3: num_samples > 1 .* need seed="),
    (BestOfRequest(_req(top_k=1, num_beams=2), 2), "request 3: num_beams > 1 cannot be combined with num_samples"),
    (BestOfRequest(_req(seed=1, num_beams=2), 2), "request 3: num_beams > 1 ranks by the AR log-likelihood"),
])
def test_best_of_argument_errors(item, what):
    with pytest.raises(ValueError, match=what):
        _stream_draws(3, item, 8, 4, False)


def test_best_of_on_fp8_and_at_the_slot_count():
    assert len(_stream_draws(0, BestOfRequest(_req(seed=1, top_k=5), 4), 8, 4, True)[1]) == 4   # n == slots runs
    with pytest.raises(ValueError, match="request 0: .*FP8"):
        _stream_draws(0, _req(num_beams=2), 8, 4, True)


def test_best_of_request_coercion():
    r = _req(seed=5, top_k=3)
    # a BestOfRequest is a tuple too: it must not be read as StreamRequest(*item)
    b = _as_request(BestOfRequest(tuple(r), 3))
    assert isinstance(b, BestOfRequest) and isinstance(b.request, StreamRequest) and b.num_samples == 3
    assert b.request.seed == 5 and b.request.top_k == 3 and b.request.num_beams == 1
    assert _as_request(tuple(r[:9])) == r._replace(num_beams=1)
    assert _as_request(r) == r
    items = [r, BestOfRequest(r, 2), tuple(r)]
    assert [_as_request(x) for x in items] == list(_as_request(x) for x in iter(items))


def test_candidates_release_siblings_first_and_the_parent_last():
    c = _Candidates(7, 4, parent=2, best_of=True)
    c.running.update([2, 3, 4, 5])
    assert c.stop(3) == [3]              # a sibling: its own slot
    assert c.stop(2) == []               # the parent: held while candidates 4 and 5 read its prompt prefix
    assert c.stop(5) == [5]
    assert c.stop(4) == [4, 2]           # the last candidate frees the parent with it
    c = _Candidates(1, 3, parent=0, best_of=True)
    c.running.update([0, 1, 2])
    assert c.stop(1) == [1] and c.stop(2) == [2] and c.stop(0) == [0]   # the parent stopping last frees itself
    c = _Candidates(1, 3, parent=None, best_of=True)                     # no shared prefix (FP8): freed one by one
    c.running.update([4, 5, 6])
    assert c.stop(5) == [5] and c.stop(4) == [4] and c.stop(6) == [6]


def test_candidates_result_shapes():
    c = _Candidates(3, 2, parent=0, best_of=True)
    for j in range(2):
        assert c.done(j, torch.full((4 + j, 8), j), torch.tensor(-1.5 - j)) == (j == 1)
    idx, codes, sc = c.result(True)
    assert idx == 3 and [x.shape[0] for x in codes] == [4, 5] and sc.tolist() == [-1.5, -2.5]
    assert c.result(False)[1] is c.codes
    p = _Candidates(4, 1)
    assert p.done(0, torch.zeros(3, 8), torch.tensor(-2.0))
    assert p.result(True)[2].shape == (1,) and torch.equal(p.result(False)[1], torch.zeros(3, 8))
    b = _Candidates(5, 1, beam=True)
    b.done(0, torch.zeros(3, 8), torch.tensor(-3.0))
    assert b.result(True)[2].shape == ()


def test_scheduler_model_keeps_fifo_and_holds_parents():
    """A host model of the stream's slots: requests of widths 1 (plain), 3 (best-of, shared prefix) and 2 (best-of)
    in 5 slots; candidates stop in a fixed order.  A parent is never handed out while a candidate of its request
    still decodes, a sibling's slot is reused while its parent decodes, and admission stays first in, first out."""
    widths = [3, 1, 2, 1, 3, 1]
    queue = list(range(len(widths)))
    free = list(range(5))
    running = {}                         # slot -> (request, candidates)
    reqs = {}
    order = []
    reused_while_parent_decodes = False
    held = set()

    def admit():
        nonlocal reused_while_parent_decodes
        taken = _take_slots(free, [widths[q] for q in queue])
        for q, ss in zip(list(queue), taken):
            c = _Candidates(q, len(ss), parent=ss[0] if len(ss) > 1 else None, best_of=len(ss) > 1)
            for s in ss:
                assert s not in held, "a held parent was handed out"
                reused_while_parent_decodes |= any(s not in r.running and r.parent in r.running
                                                   and s in sib for r, sib in sibs.values())
                c.running.add(s)
                running[s] = c
            reqs[q] = c
            sibs[q] = (c, ss[1:])
            order.append(q)
        del queue[:len(taken)]

    sibs = {}
    admit()
    # stop one candidate per round: the highest running slot first, so that parents (first slots) outlive siblings
    # in one request and are outlived in the next
    rnd = 0
    while running:
        s = max(running) if rnd % 2 == 0 else min(running)
        c = running.pop(s)
        freed = c.stop(s)
        if s == c.parent and c.running:
            held.add(s)
        for f in freed:
            held.discard(f)
        free.extend(freed)
        free.sort()
        admit()
        rnd += 1
    assert order == sorted(order) == list(range(len(widths)))
    assert sorted(free) == list(range(5)) and not held
    assert reused_while_parent_decodes
