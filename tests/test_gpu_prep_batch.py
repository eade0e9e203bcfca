"""Edges of the shared-memory raw column counts (k_col_counts_smem) and of the entry-parallel transpose: a 16-bit counter
that reaches 2^15 inside one CTA, column spaces at and one word past the shared-memory fit (past it, the replicated-copy
path counts), a rejected column id on either path, and trains whose matrices are cut into several batched launches with
empty matrices and both paths among them."""
import numpy as np
import pytest
import torch

import sampler_ref as sr
import sampler_shapes as shp
import universal_recommender_b200 as ur
from universal_recommender_b200 import _native as N
from test_gpu_sampler import assert_downsample, assert_train

pytestmark = pytest.mark.gpu


def smem_fit_cols():
    """the largest n_cols whose 16-bit counters fit one CTA's opt-in shared memory (two counters per 4-byte word)"""
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin // 4 * 2


def test_counter_reaches_2_15_inside_a_cta(ctx, orc):
    """300 000 rows all holding column 0 (and a few column 1): each CTA counts about 60 000 entries of one column, so
    every CTA hands 2^15 to the global count once before its final flush"""
    n = 300_000
    rows = [[0, 1] if r % 1000 == 0 else [0] for r in range(n)]
    mat = shp.csr(rows, 2)
    want = sr.prepare(*mat, 10, 3, 0)
    assert want.raw[0] == n and want.raw[1] == n // 1000
    assert_downsample(ctx, orc, mat, 10, 3, 0, "one hot column")
    assert_downsample(ctx, orc, mat, 10, 3, ur.FLAG_ASSUME_CANONICAL, "one hot column, verdict path")


@pytest.mark.parametrize("extra", [0, 1, 2], ids=["fit", "fit_plus_1_col", "one_word_past"])
def test_column_space_at_the_shared_memory_fit(ctx, orc, extra):
    """n_cols = the fit, one column more (same word count when the fit is even: fits), and one word past (replicated
    copies); the largest id and a hot column are used"""
    n_cols = smem_fit_cols() + extra
    rows = []
    for r in range(6000):
        row = {n_cols - 1, (r * 7919) % n_cols} if r % 3 else {1}
        rows.append(sorted(row))
    mat = shp.csr(rows, n_cols)
    for flags in (0, ur.FLAG_ASSUME_CANONICAL):
        assert_downsample(ctx, orc, mat, 5, 11, flags, f"n_cols={n_cols} flags={flags}")


@pytest.mark.parametrize("n_cols", [700, 1 << 17], ids=["shared", "copies"])
def test_column_id_outside_the_space_is_rejected(ctx, n_cols):
    """a caller-promised canonical matrix with an id = n_cols fails the call on either counting path"""
    rows = [[1, 2], [3], [], [n_cols - 1]] * 50
    rows[77] = [5, n_cols]
    nr, nc, rp, ci = shp.csr(rows, n_cols)
    with pytest.raises(N.CcoInvalidArgument):
        ctx.debug_downsample(nr, nc, rp, ci, 10, 1, ur.FLAG_ASSUME_CANONICAL)


def empty(n_rows, n_cols):
    return shp.csr([[] for _ in range(n_rows)], n_cols)


def test_train_over_several_batches_with_empty_matrices(ctx, orc):
    """eleven matrices (two batched launches of the shared-memory counts), empty ones at a batch's first, middle and last
    segment, one past the shared-memory fit between them; every indicator against the reference train"""
    base = shp.row_lengths()
    nr, nc = base[0], base[1]
    big = shp.last_column(nr, smem_fit_cols() + 2)
    mats = [base, empty(nr, 50), base, big, empty(nr, 1),
            shp.sized(nr, 3 * nr, 900, 6), empty(nr, 300), big, base, empty(nr, 7), shp.sized(nr, 2 * nr, 40, 8)]
    params = [(40, 100, None)] + [(m, 100, None) for m in (20, 30, 7, 1, 25, 5, 60, 40, 3, 9)]
    assert_train(ctx, orc, mats, params, 42, ur.FLAG_ASSUME_CANONICAL, "11 matrices canonical")
    assert_train(ctx, orc, mats, params, -1, ur.FLAG_ROWRATE_INTDIV, "11 matrices validated")
