"""The live form of the IMU ring (rebvo_b200/csrc/imu_filter.h, ImuBuffer::init_live / push, the ring of
rb_pipeline_set_imu_live) against the reference's own ImuGrabber(list_size, tsamp) (src/UtilLib/imugrabber.cpp, unmodified,
in oracle/_ref/libref_imu_grabber.so): random sequences of pushes and grabs through ring wrap-around, windows that end
exactly on a sample (the 1e-12 rule) and windows that start before the first sample.  Runs on the CPU."""
import ctypes as C

import numpy as np
import pytest

TS = 0.005


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def libs(built):
    from oracle import ref_live_imu
    from rebvo_b200 import capi
    if not ref_live_imu.available():
        pytest.skip("oracle/_ref/libref_imu_grabber.so not built (need the reference sources)")
    L = C.CDLL(capi.LIB_PATH)
    L.rb_hostmath_imu_ring_new.restype = C.c_void_p
    L.rb_hostmath_imu_ring_new.argtypes = [C.c_int, C.c_double]
    L.rb_hostmath_imu_ring_free.argtypes = [C.c_void_p]
    L.rb_hostmath_imu_ring_push.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.rb_hostmath_imu_ring_covers.argtypes = [C.c_void_p, C.c_double, C.c_double]
    L.rb_hostmath_imu_ring_grab.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p]
    L.rb_hostmath_imu_ring_state.argtypes = [C.c_void_p, C.c_void_p]
    return L, ref_live_imu


class Ring:
    """The product's live ring (hostmath exports of ImuBuffer)."""

    def __init__(self, L, list_size, tsample):
        self.L, self.h = L, L.rb_hostmath_imu_ring_new(list_size, tsample)

    def push(self, rows):
        rows = np.ascontiguousarray(rows, np.float64).reshape(-1, 7)
        return bool(self.L.rb_hostmath_imu_ring_push(self.h, _p(rows), len(rows)))

    def covers(self, t0, t1):
        return bool(self.L.rb_hostmath_imu_ring_covers(self.h, t0, t1))

    def grab(self, t0, t1):
        out = np.zeros(23)
        self.L.rb_hostmath_imu_ring_grab(self.h, t0, t1, _p(out))
        return out

    def state(self):
        """(write_inx, read_inx, size, free slots)"""
        out = np.zeros(4, np.int32)
        self.L.rb_hostmath_imu_ring_state(self.h, _p(out))
        return tuple(int(v) for v in out)

    def close(self):
        self.L.rb_hostmath_imu_ring_free(self.h)


def _samples(rng, n, t0=0.0):
    t = t0 + np.arange(n) * TS
    g = rng.normal(0, 0.6, (n, 3))
    a = rng.normal(0, 3, (n, 3)) + np.array([0, -9.8, 0])
    return np.concatenate([t[:, None], g, a], axis=1)


def _replay(ref_mod, list_size, log):
    """A fresh reference grabber that has seen the operations in log."""
    g = ref_mod.Grabber(list_size, TS)
    for op, *args in log:
        if op == "push":
            assert g.push(args[0]) == len(args[0])
        else:
            g.grab(*args)
    return g


def _tend(rng, smp, t_prev, list_size):
    """The end of the next window: past t_prev, often on a sample (exactly, within 1e-12 below it, or just outside the rule).
    A window and the sample past it fit in the ring (a longer one could never be covered)."""
    k = int(np.searchsorted(smp[:, 0], t_prev, side="right")) + int(rng.integers(0, max(1, min(14, list_size - 3))))
    k = min(k, len(smp) - 1)
    ts = smp[k, 0]
    kind = int(rng.integers(0, 5))
    t = [ts, ts - 5e-13, ts - 2e-12, ts + 0.3 * TS, ts - 0.5 * TS][kind]
    return max(t, t_prev + 1e-9)


@pytest.mark.parametrize("list_size,seed", [(4, 0), (7, 1), (16, 2), (50, 3)])
def test_live_ring_matches_reference(libs, list_size, seed):
    L, ref_mod = libs
    rng = np.random.default_rng(seed)
    smp = _samples(rng, 600)
    ours, ref = Ring(L, list_size, TS), ref_mod.Grabber(list_size, TS)
    log = []
    nxt, t_prev = 0, -0.5 * TS - 1.0   # the first window starts before the first sample
    grabs = overflows = empties = wraps = 0
    try:
        for step in range(900):
            if nxt >= len(smp):
                break
            if rng.random() < 0.55:   # push a chunk
                chunk = smp[nxt:nxt + int(rng.integers(1, list_size + 3))]
                before = ours.state()
                if ours.push(chunk):
                    assert ref.push(chunk) == len(chunk), "the reference overflowed where the ring did not (step %d)" % step
                    log.append(("push", chunk))
                    wraps += ours.state()[0] < before[0]
                    nxt += len(chunk)
                else:   # all or nothing: nothing stored; the reference stores exactly the free slots, then throws
                    overflows += 1
                    assert ours.state() == before
                    assert before[3] < len(chunk)
                    probe = _replay(ref_mod, list_size, log)
                    assert probe.push(chunk) == before[3], step
                    probe.close()
            else:   # grab the next frame's window
                t_end = _tend(rng, smp, t_prev, list_size)
                before = ours.state()
                if ours.covers(t_prev, t_end):
                    a, b = ours.grab(t_prev, t_end), ref.grab(t_prev, t_end)
                    assert a[0] > 0
                    assert a.tobytes() == b.tobytes(), (step, a, b)
                    log.append(("grab", t_prev, t_end))
                    t_prev = t_end
                    grabs += 1
                else:   # an empty window: reported (n = 0) with no change; the reference finds nothing either
                    empties += 1
                    a = ours.grab(t_prev, t_end)
                    assert a[0] == 0 and ours.state() == before
                    probe = _replay(ref_mod, list_size, log)
                    assert probe.grab(t_prev, t_end)[0] == 0, step
                    probe.close()
    finally:
        ours.close()
        ref.close()
    print("list_size %d: %d grabs, %d overflows, %d empty windows, %d wraps" % (list_size, grabs, overflows, empties, wraps))
    assert grabs >= 20 and empties >= 1 and wraps >= 1
    assert overflows >= 1 or list_size >= 50


def test_window_ending_on_a_sample(libs):
    """The 1e-12 rule: a sample at most 1e-12 past the window's end belongs to it, one further out does not."""
    L, ref_mod = libs
    smp = _samples(np.random.default_rng(9), 40, t0=1.0)
    for d, want_last in ((0.0, 20), (-5e-13, 20), (-2e-12, 19)):
        ours, ref = Ring(L, 64, TS), ref_mod.Grabber(64, TS)
        try:
            assert ours.push(smp) and ref.push(smp) == len(smp)
            t_end = smp[20, 0] + d
            a, b = ours.grab(0.5, t_end), ref.grab(0.5, t_end)   # (starts before the first sample)
            assert a.tobytes() == b.tobytes()
            assert a[0] == want_last + 1
            assert ours.state()[1] == want_last   # the last sample grabbed stays taken
        finally:
            ours.close()
            ref.close()


def test_uncovered_until_a_sample_reaches_the_end(libs):
    """A window whose end lies past the newest sample is not covered; one more sample at or past it covers it."""
    L, _ = libs
    smp = _samples(np.random.default_rng(4), 30)
    ours = Ring(L, 32, TS)
    try:
        assert ours.push(smp[:10])
        t_end = smp[10, 0] - 1e-6
        assert not ours.covers(-1.0, t_end)
        assert not ours.covers(smp[9, 0], smp[9, 0] + 1e-3)   # nothing after the start
        st = ours.state()
        assert ours.grab(-1.0, t_end)[0] == 0 and ours.state() == st
        assert ours.push(smp[10:11])
        assert ours.covers(-1.0, t_end)
        assert ours.grab(-1.0, t_end)[0] == 10
    finally:
        ours.close()
