"""CPU side of the string ingest: encode_ids / decode_ids (the offsets + bytes layout cco_ingest_strings takes and
cco_dataset_dictionary returns) and the keep=True plumbing of CcoContext.train_dataset, against a stub library."""
import ctypes as C

import numpy as np

import universal_recommender_b200 as ur
from universal_recommender_b200.similarity_analysis import CcoContext


def test_encode_ids_ascii_round_trip():
    ids = ["u1", "u10", "", "user-42", "\x00ctl\x1f", "\"q\"\\"]
    off, data = ur.encode_ids(ids)
    assert off.dtype == np.int64 and data.dtype == np.uint8
    assert off.tolist() == [0, 2, 5, 5, 12, 17, 21]
    assert bytes(data) == "".join(ids).encode()
    assert ur.decode_ids(off, bytes(data)) == ids


def test_encode_ids_multibyte_utf8():
    ids = ["é", "日本語", "a", "", "🙂x"]
    off, data = ur.encode_ids(ids)
    enc = [x.encode("utf-8") for x in ids]
    assert np.diff(off).tolist() == [len(b) for b in enc]
    assert bytes(data) == b"".join(enc)
    assert ur.decode_ids(off, bytes(data)) == ids


def test_encode_ids_empty_inputs():
    off, data = ur.encode_ids([])
    assert off.tolist() == [0] and len(data) == 0
    assert ur.decode_ids(off, b"") == []
    off, data = ur.encode_ids(["", "", ""])
    assert off.tolist() == [0, 0, 0, 0] and len(data) == 0
    assert ur.decode_ids(off, b"") == ["", "", ""]


def test_encode_ids_accepts_any_sequence():
    off, data = ur.encode_ids(x for x in ("a", "bc"))
    assert off.tolist() == [0, 1, 3] and bytes(data) == b"abc"


class _StubLib:
    """the result-side entry points of the library, answering for one 2-row, 3-cell indicator"""

    def __init__(self):
        self.rp = np.array([0, 1, 3], dtype=np.int64)
        self.ci = np.array([2, 0, 1], dtype=np.int32)
        self.ll = np.array([3.0, 2.0, 1.0], dtype=np.float64)
        self.cn = np.array([4, 5, 6], dtype=np.int32)
        self.freed, self.trained = [], []

    def cco_train_dataset(self, h, ds, params, seed, flags, out):
        self.trained.append((ds, params[0].top_k, seed.value, flags))
        out._obj.value = 0x1000
        return 0

    def cco_result_row_range(self, res, i, rb, re_):
        rb._obj.value, re_._obj.value = 0, 2
        return 0

    def cco_result_matrix(self, res, i, nr, nc, prp, pci, pll, pcn):
        nr._obj.value, nc._obj.value = 2, 3
        prp._obj.contents = C.c_int64.from_buffer(self.rp)
        pci._obj.contents = C.c_int32.from_buffer(self.ci)
        pll._obj.contents = C.c_double.from_buffer(self.ll)
        pcn._obj.contents = C.c_int32.from_buffer(self.cn)
        return 0

    def cco_result_stats(self, res, st):
        return 0

    def cco_result_free(self, res):
        self.freed.append(res.value)
        return 0


def _stub_context():
    ctx = object.__new__(CcoContext)
    ctx._L, ctx._h, ctx.last_stats, ctx._pinned_addr = _StubLib(), None, None, {}
    return ctx


def test_train_dataset_keep_returns_views_and_a_handle():
    ctx = _stub_context()
    L = ctx._L
    res, h = ctx.train_dataset((C.c_void_p(7), 1), [(500, 20, None)], seed=3, keep=True)
    (ds, top_k, seed, flags), = L.trained
    assert (ds.value, top_k, seed, flags) == (7, 20, 3, 0)
    assert L.freed == []                              # the result lives until free_result
    (rb, re_, nc, rp, ci, ll, cn), = res
    assert (rb, re_, nc) == (0, 2, 3)
    assert np.shares_memory(rp, L.rp) and np.shares_memory(ci, L.ci) and np.shares_memory(ll, L.ll)
    assert ci.tolist() == [2, 0, 1] and cn.tolist() == [4, 5, 6]
    ctx.free_result(h)
    assert L.freed == [0x1000]


def test_train_dataset_default_copies_and_frees():
    ctx = _stub_context()
    L = ctx._L
    (rb, re_, nc, rp, ci, ll, cn), = ctx.train_dataset((C.c_void_p(7), 1), [(500, 20, None)], seed=3)
    assert L.freed == [0x1000]
    assert not np.shares_memory(rp, L.rp) and not np.shares_memory(ci, L.ci)
    assert rp.tolist() == [0, 1, 3] and ll.tolist() == [3.0, 2.0, 1.0]
