"""CPU checks of beam requests in the continuous-batching stream: the first-in first-out slot choice (_take_slots) and
the StreamRequest record's new trailing field."""
import itertools
import random

import torch

from valle_b200.engine import StreamRequest, _take_slots


def test_single_requests_take_the_lowest_free_slots():
    free = [0, 2, 3, 5, 6, 7]
    assert _take_slots(free, [1, 1, 1]) == [[0], [2], [3]]
    assert free == [5, 6, 7]


def test_groups_take_the_lowest_contiguous_run():
    free = [0, 2, 3, 5, 6, 7, 9]
    assert _take_slots(free, [3]) == [[5, 6, 7]]
    assert free == [0, 2, 3, 9]
    free = [1, 3, 4, 6, 7, 8, 9]
    assert _take_slots(free, [2, 1, 2]) == [[3, 4], [1], [6, 7]]
    assert free == [8, 9]


def test_a_group_without_a_run_waits_and_so_do_the_requests_behind_it():
    free = [0, 2, 4, 6]
    assert _take_slots(free, [2, 1, 1]) == []      # four free slots, no two adjacent: nobody overtakes the group
    assert free == [0, 2, 4, 6]
    free = [0, 1, 3, 4, 5]
    assert _take_slots(free, [1, 4, 1]) == [[0]]    # the group waits for four in a row
    assert free == [1, 3, 4, 5]
    assert _take_slots([0, 1], [3]) == []


def test_progress_once_every_slot_is_free():
    rng = random.Random(0)
    for n_slots in (1, 3, 16, 64):
        for _ in range(50):
            widths = [rng.choice([1, 1, 2, 3, 4, 16]) for _ in range(rng.randint(1, 8))]
            widths = [w for w in widths if w <= n_slots] or [1]
            free = list(range(n_slots))
            taken = _take_slots(free, widths)
            assert len(taken) >= 1
            # the admitted prefix, in order, each a run; the slots are distinct and what is left stays free
            assert [len(t) for t in taken] == widths[:len(taken)]
            for t in taken:
                assert t == list(range(t[0], t[0] + len(t)))
            used = list(itertools.chain(*taken))
            assert sorted(used + free) == list(range(n_slots)) and free == sorted(free)
            if len(taken) < len(widths):   # the next one really found no run
                w = widths[len(taken)]
                assert not any(free[i + w - 1] == free[i] + w - 1 for i in range(len(free) - w + 1))


def test_stream_request_from_a_nine_field_tuple():
    t = (torch.zeros(3, dtype=torch.int64), torch.zeros((4, 8), dtype=torch.int64), None, 5, 3, 0.9, 40, 0.8,
         (10, 0.2))
    r = StreamRequest(*t)
    assert r.num_beams == 1 and r.ras == (10, 0.2) and r.top_p == 0.8 and r.seed == 5
    assert StreamRequest(*t[:2], num_beams=4).num_beams == 4
    assert StreamRequest._fields[-1] == "num_beams"
