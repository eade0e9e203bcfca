"""The key-path ingest rule (intern_ref.ingest_keys) equals Preparator.prepare on the strings the keys stand for, whatever
the key numbering: the rule the device's key-path ingest of an interned event log is held to."""
import random

import numpy as np
import pytest

from intern_ref import ingest_keys
from universal_recommender_b200 import preparator


def intern(columns, rng):
    """the keys of the strings of every column, numbered in a shuffled order (numbering is internal to the log)"""
    distinct = sorted({s for col in columns for s in col})
    rng.shuffle(distinct)
    key = {s: k for k, s in enumerate(distinct)}
    return [np.array([key[s] for s in col], np.int64) for col in columns], distinct


def check(actions, min_events, seed=0):
    rng = random.Random(seed)
    ukeys, users = intern([[u for u, _ in pairs] for _, pairs in actions], rng)
    ikeys, items = intern([[i for _, i in pairs] for _, pairs in actions], rng)
    got_users, got_items, got_mats = ingest_keys(list(zip(ukeys, ikeys)), len(users), len(items), min_events)
    want = preparator.prepare(actions, min_events)
    assert [users[k] for k in got_users] == list(want[0][1].row_ids.inverse)
    for t, (_, ds) in enumerate(want):
        assert [items[k] for k in got_items[t]] == list(ds.column_ids.inverse)
        assert np.array_equal(got_mats[t][0], ds.row_ptr)
        assert np.array_equal(got_mats[t][1], ds.col_idx)


def random_actions(seed: int, n_types: int = 3, n: int = 200):
    rng = random.Random(seed)
    out = []
    for t in range(n_types):
        # secondary types draw from a wider user pool: some of their users never act in the primary type
        pool = 30 if t == 0 else 45
        pairs = [(f"u{rng.randint(0, pool)}", f"i{rng.randint(0, 25)}") for _ in range(rng.randint(0, n))]
        pairs += [rng.choice(pairs) for _ in range(len(pairs) // 3)] if pairs else []   # repeated pairs
        rng.shuffle(pairs)
        out.append((f"e{t}", pairs))
    return out


@pytest.mark.parametrize("min_events", [0, 1, 2, 3])
@pytest.mark.parametrize("seed", range(12))
def test_random_columns(seed, min_events):
    check(random_actions(seed), min_events, seed)


@pytest.mark.parametrize("min_events", [0, 1, 2, 3])
def test_edges(min_events):
    primary = [("a", "x"), ("a", "x"), ("b", "y"), ("a", "z"), ("c", "x"), ("b", "y")]
    only_strangers = [("s1", "q"), ("s2", "r")]
    check([("buy", primary), ("view", only_strangers), ("like", [("a", "w"), ("s1", "w"), ("c", "v")])], min_events)
    check([("buy", []), ("view", [("a", "x")])], min_events)     # an empty primary type
    check([("buy", primary), ("view", [])], min_events)          # an empty secondary type
    check([("buy", [("a", "x")]), ("view", [("a", "y")])], min_events)


def test_every_user_filtered_out():
    check([("buy", [("a", "x"), ("b", "y"), ("a", "z")]), ("view", [("a", "x"), ("b", "w")])], 3)
