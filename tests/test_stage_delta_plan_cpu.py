"""CPU-only: the plan of the delta staging (arroy_b200_stage_delta_plan: which resident row every new row keeps) against a
dictionary-based restatement, and the rules of the host mirror's residency record as far as they show without a device."""
import numpy as np
import pytest

import arroy_b200 as ab

U32 = 2**32 - 1


def plan_by_dict(old_ids, new_ids, changed_ids):
    row_of = {int(i): r for r, i in enumerate(old_ids)}
    changed = {int(i) for i in changed_ids}
    return [row_of[int(i)] if int(i) in row_of and int(i) not in changed else -1 for i in new_ids]


def check(old_ids, new_ids, changed_ids):
    src, n_upload = ab.stage_delta_plan(old_ids, new_ids, changed_ids)
    want = plan_by_dict(old_ids, new_ids, changed_ids)
    assert src.tolist() == want
    assert n_upload == want.count(-1)
    kept = [s for s in want if s >= 0]
    assert kept == sorted(set(kept))   # old row -> new row is strictly increasing: what the in-place move relies on
    return want


CASES = {
    "both_empty": ([], [], []),
    "nothing_resident": ([], [1, 2, 3], []),
    "everything_deleted": ([1, 2, 3], [], [1, 2, 3]),
    "disjoint": ([1, 3, 5], [0, 2, 4, 6], []),
    "identical": ([0, 1, 2, 9], [0, 1, 2, 9], []),
    "identical_all_changed": ([0, 1, 2, 9], [0, 1, 2, 9], [0, 1, 2, 9]),
    "deletions_only": (list(range(10)), [0, 1, 4, 5, 9], [2, 3, 6, 7, 8]),
    "appends_only": (list(range(5)), list(range(9)), [5, 6, 7, 8]),
    "appends_not_listed": (list(range(5)), list(range(9)), []),
    "insert_front": ([10, 11, 12], [1, 2, 10, 11, 12], [1, 2]),
    "interleaved": ([1, 2, 4, 6, 8, 9, 12], [0, 2, 3, 4, 8, 10, 11, 12, 13], [0, 1, 3, 6, 9, 10, 11, 13]),
    "replaced": ([1, 2, 3, 4], [1, 2, 3, 4], [2, 4]),
    "changed_names_absent_ids": ([1, 2, 3], [1, 2, 3], [0, 5, 7, U32]),
    "near_u32_max": ([U32 - 3, U32 - 1, U32], [0, U32 - 3, U32 - 2, U32], [U32 - 2, U32 - 1]),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_plan_matches_the_dictionary_restatement(name):
    check(*CASES[name])


def test_plan_of_named_cases_by_hand():
    assert check(*CASES["deletions_only"]) == [0, 1, 4, 5, 9]
    assert check(*CASES["appends_not_listed"]) == [0, 1, 2, 3, 4, -1, -1, -1, -1]
    assert check(*CASES["replaced"]) == [0, -1, 2, -1]
    assert check(*CASES["near_u32_max"]) == [-1, 0, -1, 2]


@pytest.mark.parametrize("seed", range(6))
def test_plan_on_random_updates(seed):
    r = np.random.default_rng(seed)
    universe = np.unique(np.concatenate([r.integers(0, 5000, size=3000), r.integers(U32 - 500, U32 + 1, size=200)])).astype(np.uint32)
    old = np.sort(r.choice(universe, size=universe.size * 2 // 3, replace=False))
    new = np.sort(r.choice(universe, size=universe.size * 2 // 3, replace=False))
    changed = np.sort(r.choice(universe, size=universe.size // 10, replace=False))
    check(old, new, changed)


def test_no_residency_record_without_a_device():
    # the record is made when items are staged; builds that stay on the host (one Descendants node) make none, and writes to
    # the table never create one
    env = ab.Env()
    assert env.resident() is None
    w = ab.Writer(env, 0, 3, "euclidean")
    w.add_item(0, [0.0, 1.0, 2.0])
    w.add_item(1, [1.0, 1.0, 2.0])
    assert env.resident() is None
    w.builder(ab.StdRng.from_seed(bytes([42] * 32))).build()
    assert env.resident() is None
    w.del_item(0)
    w.clear()
    env.put_raw(bytes([0, 0, 3, 0, 0, 0, 1, 0]), bytes(1 + 4 + 12))
    ab.Writer(env, 0, 4, "cosine")
    assert env.resident() is None
