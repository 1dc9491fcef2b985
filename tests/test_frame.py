"""Top-level framing of EventBatch bytes (nerrf_trace_frame, csrc/ingest.cu): the host half of the live device decoder.
Host code: runs on the CPU box."""
import re

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from nerrf_b200 import ingest
from nerrf_b200._lib import NerrfError
from test_ingest import _random_batch

pytestmark = pytest.mark.usefixtures("lib_built")


def _varint(b, p):
    v, s = 0, 0
    while True:
        c = b[p]; p += 1
        v |= (c & 0x7f) << s; s += 7
        if not c & 0x80:
            return v, p


def _hop(b):
    """the top-level walk in Python: (rec_at, body_off, body_len) of every Event record"""
    out, p = [], 0
    while p < len(b):
        at = p
        tag, p = _varint(b, p)
        assert tag & 7 == 2
        n, p = _varint(b, p)
        if tag >> 3 == 1:
            out.append((at, p, n))
        p += n
    return out


def _offset(msg):
    return int(re.search(r"byte offset (\d+)", str(msg)).group(1))


@pytest.mark.parametrize("n,rich,seed", [(0, False, 0), (1, False, 1), (200, False, 2), (300, True, 3)])
def test_frame_offsets_equal_a_python_hop(n, rich, seed):
    wire = _random_batch(np.random.default_rng(seed), n, rich).SerializeToString()
    wire = wire + b"\x12\x03abc" + wire                         # an unknown length-delimited top-level field is skipped
    rec_at, body_off, body_len, consumed = ingest.frame_event_batch(wire)
    want = _hop(wire)
    assert consumed == len(wire) and len(rec_at) == len(want) == 2 * n
    assert [tuple(int(v) for v in r) for r in zip(rec_at, body_off, body_len)] == want


def test_cut_off_tail_is_carried_in_partial_mode():
    wire = _random_batch(np.random.default_rng(7), 40).SerializeToString()
    recs = _hop(wire)
    ends = [o + n for _, o, n in recs]
    for cut in (1, 2, 5, len(wire) // 2, len(wire) - 1):
        rec_at, _, _, consumed = ingest.frame_event_batch(wire[:cut], partial=True)
        whole = [e for e in ends if e <= cut]
        assert consumed == (whole[-1] if whole else 0) and len(rec_at) == len(whole)
        with pytest.raises(NerrfError, match="malformed EventBatch at byte offset %d" % consumed):
            ingest.frame_event_batch(wire[:cut])
    assert ingest.frame_event_batch(b"", partial=True)[3] == 0


def test_malformed_input_gives_the_host_decoder_offset():
    wire = _random_batch(np.random.default_rng(6), 4).SerializeToString()
    for bad in (wire + b"\x0a\xff\xff\xff\xff\xff\xff\xff\xff\xff\xff\xff",      # 11-byte length varint
                wire + b"\x0b\x00",                                              # group wire type
                wire[:-3]):
        with pytest.raises(NerrfError) as e_dec:
            ingest.decode_event_batch(bad)
        for partial in (False, True):
            if partial and bad == wire[:-3]:
                continue                                                         # merely cut off: not an error there
            with pytest.raises(NerrfError) as e_fr:
                ingest.frame_event_batch(bad, partial=partial)
            assert _offset(e_fr.value) == _offset(e_dec.value)


@settings(max_examples=200, deadline=None)
@given(st.binary(max_size=200))
def test_fuzz_framing_agrees_with_the_decoder(data):
    """the decoder's verdict = framing, then the Event bodies: its error offset is the framing error or a framed record"""
    try:
        cols = ingest.decode_event_batch(data)
        dec = None
    except NerrfError as e:
        cols, dec = None, _offset(e)
    try:
        rec_at, _, _, consumed = ingest.frame_event_batch(data)
        fr = None
    except NerrfError as e:
        fr = _offset(e)
    if fr is not None:
        assert dec is not None and dec <= fr
    else:
        assert consumed == len(data)
        if dec is None:
            assert cols.n == len(rec_at)
        else:
            assert dec in set(int(v) for v in rec_at)
