"""oracle/pop_oracle.py and model_oracle.ranking_scores (what the GPU tests of the model index trust) against
tests/popmodel_ref.py, an independent reading of PopModel.scala:113-182, on the directed shapes of
tests/popmodel_shapes.py.  Runs on every CPU box: the restatement is pinned here, and so is the power of the shapes --
a bucket edge moved by a millisecond, or an inclusive upper bound, changes a score of some shape."""
import pytest

import model_oracle as mo
import popmodel_ref as ref
import popmodel_shapes as shp
from oracle import pop_oracle as po

SHAPES = shp.shapes()
IDS = [s[0] for s in SHAPES]


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_restatements_match_the_independent_reference(shape):
    name, mode, start, end, n, items, times = shp.in_range(shape)
    want = ref.pop_model(mode, items, times, start, end)
    assert all(type(v) is int for v in want.values())
    got = po.pop_model(mode, items, times, start, end)
    assert {j: int(v) for j, v in got.items()} == want and all(float(v).is_integer() for v in got.values())
    ids = [f"id-{(j * 7 + 3) % 1009}" for j in range(n)]
    by_id = mo.ranking_scores(mode, start, end, [([ids[j] for j in items[:len(items) // 2]], times[:len(times) // 2]),
                                                 ([ids[j] for j in items[len(items) // 2:]], times[len(times) // 2:])])
    assert by_id == {ids[j]: v for j, v in want.items()}


def test_joda_intervals_of_the_reference():
    # dur 8: hot thirds are [0,2) [2,4) [4,8): the newest third takes the remainder; 2 * dur // 3 would say 5
    assert ref.edges("hot", 0, 8) == [0, 2, 4, 8]
    assert ref.edges("hot", -10, 1) == [-10, -7, -4, 1]
    assert ref.edges("trending", -3, 4) == [-3, 0, 4] and ref.edges("trending", 5, 6) == [5, 5, 6]
    assert ref.edges("popular", 3, 3) == [3, 3]
    with pytest.raises(ValueError):
        ref.Interval(2, 1)
    # by hand on [0, 90): the cases of tests/test_pop_model.py
    items = [0, 0, 0, 1, 1, 1, 1, 2, 2, 3]
    times = [5, 35, 65, 10, 50, 70, 80, 40, 89, 90]
    assert ref.pop_model("popular", items, times, 0, 90) == {0: 3, 1: 4, 2: 2}
    assert ref.pop_model("trending", items, times, 0, 90) == {0: -1, 1: 2, 2: 0}
    assert ref.pop_model("hot", items, times, 0, 90) == {0: 0, 1: 1}
    assert ref.pop_model("trending", [0, 1], [50, 60], 0, 90) == {}
    assert ref.pop_model("hot", [0, 0], [5, 70], 0, 90) == {}


def _mutant(mode, items, times, edges, upper_inclusive, rules=True):
    """the histograms over explicit edges, with the faults a kernel could have"""
    nb = len(edges) - 1
    counts = [dict() for _ in range(nb)]
    for j, t in zip(items, times):
        for b in range(nb):
            if edges[b] <= t and (t <= edges[b + 1] if upper_inclusive else t < edges[b + 1]):
                counts[b][j] = counts[b].get(j, 0) + 1
    if rules and any(not c for c in counts[:-1]):
        return {}
    weights = {1: (1,), 2: (-1, 1), 3: (1, -2, 1)}[nb]
    return {j: sum(w * c[j] for w, c in zip(weights, counts)) for j in counts[0] if all(j in c for c in counts)}


@pytest.mark.parametrize("mode", shp.MODES)
def test_every_edge_fault_changes_a_score(mode):
    """on every window that has an older bucket, each single fault is visible in that one shape"""
    checked = 0
    for name, m, start, end, n, items, times in shp.edge_shapes():
        if m != mode:
            continue
        edges = ref.edges(mode, start, end)
        want = ref.pop_model(mode, items, times, start, end)
        assert _mutant(mode, items, times, edges, False) == want, name
        if end - start < len(edges) - 1:      # no older bucket: every variant is empty too
            assert want == {} or mode == "popular", name
            continue
        checked += 1
        assert want, name
        assert _mutant(mode, items, times, edges, True) != want, name
        for k in range(len(edges)):
            for d in (-1, 1):
                moved = list(edges)
                moved[k] += d
                if all(a <= b for a, b in zip(moved, moved[1:])):
                    assert _mutant(mode, items, times, moved, False) != want, (name, k, d)
    assert checked >= 4 * (len(shp.DURATIONS) - 3)
    if mode == "hot":       # the durations with dur % 3 == 2 are where start + 2 * dur / 3 is a millisecond late
        assert any(ref.edges("hot", s, e)[2] != s + 2 * (e - s) // 3 for _, m, s, e, *_ in shp.edge_shapes() if m == "hot")


def test_rule_and_key_shapes_hold_what_their_names_promise():
    by_name = {s[0]: s for s in SHAPES}
    for mode, nb in (("trending", 2), ("hot", 3)):
        name, _, start, end, n, items, times = by_name[f"subsets-{mode}"]
        assert n == (1 << nb) - 1 and ref.pop_model(mode, items, times, start, end).keys() == {n - 1}
        for empty in range(nb):
            name, _, start, end, n, items, times = by_name[f"bucket{empty}-empty-{mode}"]
            edges = ref.edges(mode, start, end)
            assert ref.pop_model(mode, items, times, start, end) == {}
            # without the isEmpty rules the older and middle cases would still be empty only because of the join: the
            # rules show in totals, which the key shapes below exercise; here the buckets are what the name says
            filled = [any(edges[b] <= t < edges[b + 1] for t in times) for b in range(nb)]
            assert filled == [b != empty for b in range(nb)]
        name, _, start, end, n, items, times = by_name[f"scores-{mode}"]
        got = ref.pop_model(mode, items, times, start, end)
        assert len(got) == n and 0 in got.values() and min(got.values()) < 0 < max(got.values())
        # the older bucket holds out-of-range keys only: counting them into the totals would let item 1 through when the
        # item test is also missing, and the in-range result is empty
        shape = by_name[f"keys-outside-only-older-{mode}"]
        assert {-1, shape[4]} <= set(shape[5])
        _, _, start, end, n, items, times = shp.in_range(shape)
        assert ref.pop_model(mode, items, times, start, end) == {}
    for mode in shp.MODES:
        shape = by_name[f"keys-outside-{mode}"]
        assert {-1, shape[4]} <= set(shape[5])
        assert ref.pop_model(mode, *shp.in_range(shape)[5:], shape[2], shape[3]).keys() == {0, 4}
        assert len(by_name[f"grid-stride-{mode}"][5]) > 132 * 8 * 256
        assert by_name[f"hot-key-{mode}"][5][:4096] == [2] * 4096
