"""Simpler round-2 variant: integer cut on level k11 == 1 only.
  c1* = smallest colB such that at least k strongly-positive k11==1 cells have colB <= c1*   (pure integer prefix scan)
  level-1 strong cells with colB > c1* cannot be in the top-k (LLR strictly decreasing in colB) -> never evaluated;
  every other cell is evaluated as today.  Exact."""
import sys
sys.path.insert(0, __import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__)))))
from select_model import llr, brute, random_row
import bisect
import random

def level1_cut(cells, ra, N, k, min_llr, item, self_, Cmax=1024, stats=None):
    hist = [0] * Cmax
    def strong1(b, k11, cb):
        return k11 == 1 and cb < Cmax and 2 * ra * cb < N and not (self_ and b == item)
    for b, k11, cb in cells:
        if strong1(b, k11, cb): hist[cb] += 1
    cut, cum = None, 0
    for c in range(Cmax):
        cum += hist[c]
        if cum >= k:
            cut = c
            break
    out, evals = [], 0
    for b, k11, cb in cells:
        if self_ and b == item: continue
        if cut is not None and strong1(b, k11, cb) and cb > cut: continue      # integer test only
        v = llr(k11, ra, cb, N); evals += 1
        if min_llr is not None and not v >= min_llr: continue
        if v > 0: out.append((-v, b, k11))
    out.sort()
    if stats is not None:
        stats['evals'] = stats.get('evals', 0) + evals; stats['cells'] = stats.get('cells', 0) + len(cells)
    return [(b, -nv, k11) for nv, b, k11 in out[:k]]


def column_order(marg):
    """Column order of B' (k_col_order): key = rank under (colB ascending, column id ascending).
    marg: {column id: colB}.  Returns key_of_col, col_of_key, marg_key, first_key_of_cb[0 .. max colB + 1]."""
    col_of_key = sorted(marg, key=lambda b: (marg[b], b))
    key_of_col = {b: key for key, b in enumerate(col_of_key)}
    marg_key = [marg[b] for b in col_of_key]
    max_cb = max(marg_key, default=0)
    first_key_of_cb = [bisect.bisect_left(marg_key, c) for c in range(max_cb + 2)]
    return key_of_col, col_of_key, marg_key, first_key_of_cb


def key_path(cells, ra, N, k, min_llr, item, self_, stats=None, Cmax=512, levels=15):
    """k_rows after the column renumbering: the row's cells are (key, k11) words; colB only comes from marg_key[key].
    A row with 2 rowA max(colB) < N takes the key path (key cut, key-valued dominance frontier, no colB read before the
    fp64 stage); any other row keeps the colB cut (Cmax bins) and the colB frontier.  Cells are filtered and evaluated
    in the order given (the kernel's table order), against a running k-th-best threshold."""
    marg = {b: cb for b, _, cb in cells}
    if self_ and item not in marg:
        marg[item] = 1                        # the diagonal column exists in B' even when the row does not touch it
    key_of_col, col_of_key, marg_key, first_key_of_cb = column_order(marg)
    words = [(key_of_col[b], k11) for b, k11, _ in cells]
    keyed = 2 * ra * marg_key[-1] < N if marg_key else True
    diag = key_of_col[item] if self_ else -1
    cut = None
    if keyed:
        ones = sorted(key for key, k11 in words if k11 == 1 and key != diag)
        if len(ones) >= k: cut = ones[k - 1]  # exact k-th smallest key: ties in colB ordered by column id
    else:
        hist = [0] * Cmax
        for key, k11 in words:
            cb = marg_key[key]
            if k11 == 1 and key != diag and cb < Cmax and 2 * ra * cb < N: hist[cb] += 1
        cum = 0
        for c in range(Cmax):
            cum += hist[c]
            if cum >= k:
                cut = c
                break
    frontier = [float('inf')] * (levels + 1)
    best, evals = [], 0                       # best: (-llr, col) of the candidates so far, sorted
    for key, k11 in words:
        if key == diag: continue
        cb = marg_key[key]
        if keyed:
            if k11 <= levels and key >= frontier[k11]: continue
            if k11 == 1 and cut is not None and key > cut: continue
        else:
            pos_side = ra * cb < k11 * N
            if pos_side and k11 <= levels and cb >= frontier[k11]: continue
            if k11 == 1 and cut is not None and cb > cut and 2 * ra * cb < N: continue
        v = llr(k11, ra, cb, N); evals += 1
        b = col_of_key[key]
        min_ok = min_llr is None or v >= min_llr
        strict_fail = v > 0 and not min_ok
        if v > 0 and min_ok:
            if len(best) >= k and v < -best[k - 1][0]: strict_fail = True
            best.append((-v, b, k11)); best.sort()
        if strict_fail and ra * cb < k11 * N:
            f = first_key_of_cb[cb] if keyed else cb
            for kk in range(min(k11, levels), 0, -1):
                frontier[kk] = min(frontier[kk], f)
    if stats is not None:
        stats['evals'] = stats.get('evals', 0) + evals; stats['cells'] = stats.get('cells', 0) + len(cells)
        path = 'keyed' if keyed else 'fallback'
        stats[path] = stats.get(path, 0) + 1
    return [(b, -nv, k11) for nv, b, k11 in best[:k]]


def tied_row(rng):
    """A row whose k11 == 1 cells share a handful of colB values: long ties in colB around the k-th cell."""
    N = 10 ** rng.randrange(3, 8)
    ra = rng.randrange(1, max(2, min(600, N // 2)))
    values = sorted(rng.sample(range(1, min(600, N - ra) + 1), min(rng.randrange(1, 6), min(600, N - ra))))
    cells = []
    for b in rng.sample(range(5000), rng.randrange(0, 800)):
        cb = rng.choice(values)
        k11 = min(1 if rng.random() < 0.85 else rng.randrange(1, 8), ra, cb)
        if N - ra - cb + k11 < 0: continue
        cells.append((b, k11, cb))
    return cells, ra, N


if __name__ == '__main__':
    rng = random.Random(11)
    for t in range(3000):
        cells, ra, N = random_row(rng)
        k = rng.choice([1, 5, 50, 50, 200]); min_llr = rng.choice([None, None, 0.5, 5.0])
        item = rng.randrange(0, 5000); self_ = rng.random() < 0.3
        assert brute(cells, ra, N, k, min_llr, item, self_) == level1_cut(cells, ra, N, k, min_llr, item, self_), t
    print('3000 random rows identical')
