"""bag_replay.slot_queue: the scheduler that queues recordings through sequence mode's slots (bag_replay.replay,
tools/seq_bench.py and the GPU suite's drivers)."""
import numpy as np

from conftest import pkg

slot_queue = pkg("bag_replay").slot_queue


def steps(lengths, n_slots):
    return [(r.tolist(), who) for r, who in slot_queue(lengths, n_slots)]


def test_hand_worked():
    # job 1 ends after one step and slot 1 restarts with job 2; slot 0 idles once job 0 ends and nothing is left
    assert steps([2, 1, 3], 2) == [
        ([0, 0], [(0, 0), (1, 0)]),
        ([0, 1], [(0, 1), (2, 0)]),
        ([0, 0], [None, (2, 1)]),
        ([0, 0], [None, (2, 2)]),
    ]


def test_more_jobs_than_slots():
    assert steps([1, 1, 1, 1, 1], 2) == [
        ([0, 0], [(0, 0), (1, 0)]),
        ([1, 1], [(2, 0), (3, 0)]),
        ([1, 0], [(4, 0), None]),
    ]


def test_fewer_jobs_than_slots():
    assert steps([2, 1], 4) == [
        ([0, 0, 0, 0], [(0, 0), (1, 0), None, None]),
        ([0, 0, 0, 0], [(0, 1), None, None, None]),
    ]


def test_empty_jobs_are_skipped():
    # an empty job never takes a slot: the slot takes the next job on the same step, and a slot that has not run a job
    # yet is not restarted
    assert steps([1, 0, 2], 1) == [([0], [(0, 0)]), ([1], [(2, 0)]), ([0], [(2, 1)])]
    assert steps([0, 1], 1) == [([0], [(1, 0)])]
    assert steps([0, 0], 3) == []


def test_single_slot():
    assert steps([2, 2], 1) == [([0], [(0, 0)]), ([0], [(0, 1)]), ([1], [(1, 0)]), ([0], [(1, 1)])]


def test_every_step_of_every_job_once_in_order():
    rng = np.random.default_rng(3)
    for _ in range(50):
        lengths = rng.integers(0, 5, rng.integers(0, 12)).tolist()
        n_slots = int(rng.integers(1, 5))
        seen, job_of_slot, used = [[] for _ in lengths], [None] * n_slots, [False] * n_slots
        for restart, who in slot_queue(lengths, n_slots):
            assert restart.dtype == np.uint8 and len(restart) == len(who) == n_slots
            for j, w in enumerate(who):
                new = w is not None and w[0] != job_of_slot[j]
                assert restart[j] == (new and used[j]), (lengths, n_slots)
                if w is not None:
                    seen[w[0]].append(w[1])
                    job_of_slot[j], used[j] = w[0], True
        assert seen == [list(range(n)) for n in lengths], (lengths, n_slots)
