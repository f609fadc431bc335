"""CPU: tracker records (ht_tracker_export / ht_tracker_import) through the host build of the functions the kernels use
(ht_selftest_tracker_pack / _check / _unpack):

  * the lockstep of test_host_lifecycle.py (tracker_step against the oracle) over every case of the lifecycle and main
    goldens, with the stream's state packed into a record, checked and unpacked into a fresh buffer before every
    call: the events still equal the goldens, and every repack is byte-identical;
  * the layout include/headtrackr_b200.h states, and the checksum it defines;
  * every single-byte flip of a record is rejected, and so are a wrong magic, version or size and crafted records
    with a valid checksum but an out-of-range field."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

import test_host_lifecycle
from test_cascade_host import st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_host_lifecycle import ALL_CASES, TM_CS, case_id, tracker_params

HEADER = (Path(__file__).resolve().parent.parent / "include" / "headtrackr_b200.h").read_text()


def define(name):
    return int(re.search(rf"#define {name} (0x[0-9a-fA-F]+|\d+)u?\b", HEADER).group(1), 0)


R = define("HT_TRACKER_RECORD_BYTES")
MAGIC, VERSION = define("HT_TRACKER_RECORD_MAGIC"), define("HT_TRACKER_RECORD_VERSION")
STATE, PARAMS, TRACK, COST, HIST = 32, 320, 416, 464, 480      # section offsets stated in the header
# fields the import check looks at (offsets inside the record)
MODE, N_WB, N_DIAG = STATE + 0, STATE + 4, STATE + 144 + 8
ALPHA, DISTANCE = PARAMS + 8 + 16, PARAMS + 8 + 40
SW, SH, INITIALISED = TRACK + 8, TRACK + 12, TRACK + 44
REC_OK, BAD_MAGIC, BAD_VERSION, BAD_SIZE, BAD_CHECKSUM, BAD_MODE, BAD_WB, BAD_DIAG, BAD_PARAMS, BAD_TRACK = range(10)


def bind(st):
    vp = C.c_void_p
    st.ht_selftest_tracker_size.restype = C.c_int
    st.ht_selftest_tracker_params_size.restype = C.c_int
    st.ht_selftest_tracker_params.argtypes = [vp, vp]
    st.ht_selftest_tracker_pack.argtypes = [vp, vp, vp, vp, vp, vp]
    st.ht_selftest_tracker_check.argtypes = [vp]
    st.ht_selftest_tracker_unpack.argtypes = [vp, vp, vp, vp, vp, vp]
    st.ht_selftest_tracker.argtypes = [vp, C.c_int, vp, C.c_double, vp, C.c_int, vp, C.c_double, C.c_int, C.c_int, vp, vp]


def checksum(rec):
    """sum of w_i * (2i + 1) mod 2^64 over the u32 words from byte 24 on"""
    w = np.frombuffer(rec[24:].tobytes(), "<u4").astype(np.uint64)
    return int((w * (2 * np.arange(len(w), dtype=np.uint64) + 1)).sum(dtype=np.uint64))


def reseal(rec):
    rec = rec.copy()
    rec[16:24] = np.frombuffer(np.uint64(checksum(rec)).tobytes(), np.uint8)
    return rec


class Sections:
    """one stream's sections as ht_selftest_tracker_pack takes them"""

    def __init__(self, st):
        self.state = C.create_string_buffer(st.ht_selftest_tracker_size())
        self.params = C.create_string_buffer(st.ht_selftest_tracker_params_size())
        self.track = C.create_string_buffer(48)
        self.hist = np.zeros(4096, np.uint32)
        self.cost = np.zeros(2, np.int32)

    def pack(self, st):
        rec = np.zeros(R, np.uint8)
        assert st.ht_selftest_tracker_pack(self.state, self.params, self.track, self.hist.ctypes.data, self.cost.ctypes.data,
                                           rec.ctypes.data) == R
        return rec

    def unpack(self, st, rec):
        assert st.ht_selftest_tracker_unpack(rec.ctypes.data, self.state, self.params, self.track, self.hist.ctypes.data,
                                             self.cost.ctypes.data) == 0


def check(st, rec):
    return st.ht_selftest_tracker_check(np.ascontiguousarray(rec).ctypes.data)


class Migrating:
    """The host build for test_host_lifecycle's lockstep, with every call of the state machine made on a state that
    has just come out of a record: pack, check, unpack into fresh sections, repack (byte-identical)."""

    def __init__(self, st):
        bind(st)
        self._st = st
        self.ht_selftest_tracker_size = st.ht_selftest_tracker_size
        self.cur = Sections(st)
        self.rng = np.random.default_rng(3)
        self.moves, self.modes = 0, set()

        def tracker(state, op, params, *rest):
            if op != 0:
                self._move(state, params)
            mode = st.ht_selftest_tracker(state, op, params, *rest)
            seed = rest[-1]
            if op == 3 and seed[0]:       # the camshift section k_track_init writes: window, calcAngles, a model
                t = np.zeros(12, np.int32)
                t[0:4] = seed[1:5]
                t[10] = params._obj.calc_angles
                t[11] = 1
                C.memmove(self.cur.track, t.ctypes.data, 48)
                self.cur.hist[:] = self.rng.integers(0, 1 << 32, 4096, dtype=np.uint32)
                self.cur.cost[:] = self.rng.integers(1, 1 << 31, 2)
            return mode
        self.ht_selftest_tracker = tracker

    def _move(self, state, params):
        st, cur = self._st, self.cur
        C.memmove(cur.state, state, len(cur.state))
        st.ht_selftest_tracker_params(params, cur.params)
        rec = cur.pack(st)
        assert check(st, rec) == REC_OK
        fresh = Sections(st)
        fresh.unpack(st, rec)
        assert np.array_equal(fresh.pack(st), rec)                      # repack: byte-identical
        assert fresh.state.raw == cur.state.raw and fresh.params.raw == cur.params.raw
        mode = int(rec[MODE:MODE + 4].view(np.int32)[0])
        if mode == TM_CS:
            assert fresh.track.raw == cur.track.raw and np.array_equal(fresh.hist, cur.hist)
            assert np.array_equal(fresh.cost, cur.cost)
        else:                                                           # canonical form: dead camshift state is zeros
            assert not rec[TRACK:].any() and not fresh.hist.any() and not fresh.cost.any()
        C.memmove(state, fresh.state, len(fresh.state))                 # the lockstep goes on from the unpacked state
        self.cur = fresh
        self.moves += 1
        self.modes.add(mode)


@pytest.mark.parametrize("gc", ALL_CASES, ids=case_id)
def test_lockstep_through_a_record_before_every_call(st, gc, blob):
    m = Migrating(st)
    test_host_lifecycle.test_device_state_machine_replays_every_step(m, gc, blob)
    assert m.moves >= len(gc[1]["steps"]) and {1, 2, 3, TM_CS} <= m.modes


def cs_record(st):
    """a record of a stream in CS with a live camshift section"""
    bind(st)
    s = Sections(st)
    params = tracker_params({"params": {"calcAngles": True}})
    st.ht_selftest_tracker_params(C.byref(params), s.params)
    out, seed = C.create_string_buffer(512), (C.c_int32 * 5)()
    st.ht_selftest_tracker(s.state, 0, C.byref(params), 0.0, None, 0, None, 0.0, 160, 120, out, seed)
    st.ht_selftest_tracker(s.state, 1, C.byref(params), 0.0, None, 0, None, 0.0, 160, 120, out, seed)
    st.ht_selftest_tracker(s.state, 3, C.byref(params), 100.0, None, 0, None, 0.0, 160, 120, out, seed)
    state = np.frombuffer(s.state.raw, np.int32).copy()
    state[0] = TM_CS                                                    # as after a hand-off
    C.memmove(s.state, state.ctypes.data, len(s.state))
    C.memmove(s.track, np.array([10, 12, 30, 40, 25, 32, 30, 40, 0, 0, 1, 1], np.int32).ctypes.data, 48)
    rng = np.random.default_rng(11)
    s.hist[:] = rng.integers(0, 1 << 32, 4096, dtype=np.uint32)
    s.cost[:] = [57, 1234]
    return s.pack(st)


def test_layout_and_checksum(st):
    rec = cs_record(st)
    assert len(rec) == R == HIST + 4096 * 4 and R % 16 == 0
    w = rec[:16].view("<u4")
    assert (w[0], w[1], w[2], w[3]) == (MAGIC, VERSION, R, 0)
    assert rec[:4].tobytes() == b"HTR1"
    assert int(rec[16:24].view("<u8")[0]) == checksum(rec)
    assert not rec[24:STATE].any()
    assert rec[MODE:MODE + 4].view("<i4")[0] == TM_CS and rec[N_WB:N_WB + 4].view("<i4")[0] == 1
    assert rec[PARAMS + 4:PARAMS + 8].view("<i4")[0] == 1                           # calcAngles
    assert rec[ALPHA:ALPHA + 8].view("<f8")[0] == 0.35 and rec[DISTANCE:DISTANCE + 8].view("<f8")[0] == 60.0
    assert tuple(rec[TRACK:TRACK + 16].view("<i4")) == (10, 12, 30, 40)
    assert tuple(rec[COST:COST + 8].view("<i4")) == (57, 1234)
    assert rec[HIST:HIST + 16].view("<u4")[0] == np.random.default_rng(11).integers(0, 1 << 32, 4096, dtype=np.uint32)[0]
    assert check(st, rec) == REC_OK and check(st, reseal(rec)) == REC_OK


def test_every_single_byte_flip_is_rejected(st):
    rec = cs_record(st)
    for off in range(R):
        for x in (0x01, 0xFF):
            bad = rec.copy()
            bad[off] ^= x
            assert check(st, bad) != REC_OK, (off, x)


def put(rec, off, value, dtype):
    rec = rec.copy()
    rec[off:off + np.dtype(dtype).itemsize] = np.frombuffer(np.array(value, dtype).tobytes(), np.uint8)
    return rec


@pytest.mark.parametrize("off, value, dtype, code", [
    (0, 0x31525449, "<u4", BAD_MAGIC),
    (4, 2, "<u4", BAD_VERSION),
    (8, R - 16, "<u4", BAD_SIZE),
    (12, 1, "<u4", BAD_SIZE),
    (MODE, 7, "<i4", BAD_MODE),
    (MODE, -1, "<i4", BAD_MODE),
    (N_WB, 16, "<i4", BAD_WB),
    (N_WB, -1, "<i4", BAD_WB),
    (N_DIAG, -1, "<i4", BAD_DIAG),
    (N_DIAG, 7, "<i4", BAD_DIAG),
    (ALPHA, -0.01, "<f8", BAD_PARAMS),
    (ALPHA, 1.5, "<f8", BAD_PARAMS),
    (ALPHA, float("nan"), "<f8", BAD_PARAMS),
    (DISTANCE, 0.0, "<f8", BAD_PARAMS),
    (SW, 0, "<i4", BAD_TRACK),
    (SH, -3, "<i4", BAD_TRACK),
    (INITIALISED, 0, "<i4", BAD_TRACK),
])
def test_crafted_records_with_a_valid_checksum_are_rejected(st, off, value, dtype, code):
    rec = cs_record(st)
    assert check(st, put(rec, off, value, dtype)) == (BAD_CHECKSUM if off >= 24 else code)   # the checksum first
    assert check(st, reseal(put(rec, off, value, dtype))) == code


def test_edge_values_are_accepted(st):
    rec = cs_record(st)
    for off, value, dtype in [(N_WB, 15, "<i4"), (N_WB, 0, "<i4"), (N_DIAG, 6, "<i4"), (N_DIAG, 0, "<i4"),
                              (ALPHA, 0.0, "<f8"), (ALPHA, 1.0, "<f8")]:
        assert check(st, reseal(put(rec, off, value, dtype))) == REC_OK, (off, value)
    # a stream that is not in CS carries no camshift tracker: an empty window is fine there
    assert check(st, reseal(put(put(put(rec, MODE, 3, "<i4"), SW, 0, "<i4"), INITIALISED, 0, "<i4"))) == REC_OK
