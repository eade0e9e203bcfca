"""The three readers of Elasticsearch responses on one table of malformed frames: an _msearch body (cco_search_results_*),
a _search / scroll page (cco_index_pages_*) and a _bulk response (cco_index_write_*).  Each reports a frame with its own
prefix, repeats the message on the next call and on finish, and after a successful finish reports that it is finished."""
import ctypes as C

import pytest

from universal_recommender_b200 import _native as N
from universal_recommender_b200.similarity_analysis import SearchResults

pytestmark = pytest.mark.gpu

GOOD_BODY = b'{"responses":[]}'
GOOD_PAGE = b'{"hits":{"hits":[]}}'
ONE = b'{"index":{"_id":"a"}}\n{"id":"a"}\n'
GOOD_BULK = b'{"items":[{"index":{"_id":"a","status":201}}]}'

# frame -> (byte, message) after the reader's prefix, or None: the top level is not an object
FRAMES = {
    "unclosed string": (b'{"took":1,"x":"ab', (17, "a string is not closed")),
    "closing bracket with nothing open": (b'{"took":1}}', (10, "unbalanced or mismatched brackets")),
    "mismatched pair": (b'{"x":[1}}', (7, "unbalanced or mismatched brackets")),
    "trailing bytes": (b'{"x":1} x', (7, "malformed JSON")),
    "bad escape in a name": (b'{"\\q":1}', (2, "a string holds a bad escape or a raw byte < 0x20")),
    "empty body": (b"", None),
    "top-level array": (b'[{"x":1}]', None),
}


class Search:
    """cco_search_results through the C entries: body 0 is read by the next append"""
    prefix = "response body 0"
    not_object = 'response body 0, byte 0: the top level is not an object with one "responses" array'
    finished = "the results are finished"

    def __init__(self, ctx):
        self.ctx, self.L, self.h = ctx, N.lib(), C.c_void_p()
        prm = N.SearchResultsParamsT(0, None, N.SR_TEXT)
        N.check(self.L.cco_search_results_begin(ctx._h, C.byref(prm), C.byref(self.h)))

    def append(self, body):
        N.check(self.L.cco_search_results_append(self.h, body, len(body), -1, None, None, None))

    def feed(self, frame):
        self.append(frame)
        self.append(GOOD_BODY)

    def next_call(self):
        self.append(GOOD_BODY)

    def succeed(self):
        self.append(GOOD_BODY)

    def finish(self):
        out = N.SearchResultsOutT()
        N.check(self.L.cco_search_results_finish(self.h, C.byref(out)))
        SearchResults(self.ctx, out, [])   # hands the buffers back

    def free(self):
        self.L.cco_search_results_free(self.h)


class Pages:
    """cco_index_pages: page 0 is good, page 1 is the frame"""
    prefix = "page 1"
    not_object = "page 1: the top level is not an object"
    finished = "the index pages are finished"

    def __init__(self, ctx):
        self.r = ctx.index_pages()

    def feed(self, frame):
        self.r.append(GOOD_PAGE)
        self.r.append(frame)

    def next_call(self):
        self.r.append(GOOD_PAGE)

    def succeed(self):
        self.r.append(GOOD_PAGE)

    def finish(self):
        self.r.finish()

    def free(self):
        self.r.free()


class Write:
    """cco_index_write of one document: the frame is the response to request 0"""
    prefix = "request 0"
    not_object = "request 0: the top level is not an object"
    finished = "the index write is finished"

    def __init__(self, ctx):
        self.w = ctx.index_write(ONE)

    def feed(self, frame):
        self.w.response(0, frame)

    def next_call(self):
        self.w.response(0, GOOD_BULK)

    def succeed(self):
        self.w.response(0, GOOD_BULK)

    def finish(self):
        self.w.finish()

    def free(self):
        self.w.free()


READERS = {"search_results": Search, "index_pages": Pages, "index_write": Write}


def raises_exactly(call, msg):
    with pytest.raises(N.CcoInvalidArgument) as e:
        call()
    assert str(e.value) == f"[cco status {N.E_INVALID_ARG}] {msg}"


@pytest.mark.parametrize("reader", list(READERS))
@pytest.mark.parametrize("frame", list(FRAMES))
def test_malformed_frame(ctx, reader, frame):
    body, at = FRAMES[frame]
    r = READERS[reader](ctx)
    msg = r.not_object if at is None else f"{r.prefix}, byte {at[0]}: {at[1]}"
    try:
        raises_exactly(lambda: r.feed(body), msg)
        raises_exactly(r.next_call, msg)
        raises_exactly(r.finish, msg)
    finally:
        r.free()


@pytest.mark.parametrize("reader", list(READERS))
def test_call_after_finish(ctx, reader):
    r = READERS[reader](ctx)
    try:
        r.succeed()
        r.finish()
        raises_exactly(r.next_call, r.finished)
    finally:
        r.free()
