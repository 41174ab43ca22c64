"""Live IMU input (ImuMode=1: rb_pipeline_set_imu_live + rb_pipeline_push_imu) on the EuRoC-like stream with its synthetic
200 Hz samples.  With the integration step set to dataset mode's (the samples' mean spacing) the live ring gives dataset
mode's bytes, however the samples arrive: all up front, one at a time, in chunks cut at frame times, through a ring a few
frames deep, after a push the samples did not cover or a push_imu that overflowed.  With SampleTime = 0.005 it follows the
reference's own REBVO in ImuMode=1 (oracle/ref_live_imu.cpp, unmodified reference sources), on the CPU reference and on the
shim."""
import os
import re

import numpy as np
import pytest

from pipeline_util import assert_knife_edge, euroc_sequence, frames_file, push, raw, run_pipeline

pytestmark = pytest.mark.gpu
NF = 30
RB_ERR_ARG, RB_ERR_STATE = -2, -4


@pytest.fixture(scope="module")
def stream():
    from rebvo_b200 import capi, synth
    seq = euroc_sequence()
    ts, fr = seq.frames(NF)
    imu = synth.imu_samples(seq, NF)
    return capi.default_params(synth.EUROC), ts, fr, imu


def _imu_params():
    from rebvo_b200 import capi
    return capi.default_imu_params(InitBias=1, InitBiasFrameNum=5)   # (run_pipeline's)


def _dataset_tsample(imu):
    return (imu[-1, 0] - imu[0, 0]) / (len(imu) - 1)


def _code(err):
    m = re.search(r"error (-?\d+)", str(err))
    return int(m.group(1)) if m else None


def _raises(code, fn, *args):
    from rebvo_b200 import capi
    with pytest.raises(capi.RbError) as e:
        fn(*args)
    assert _code(e.value) == code, str(e.value)


class Feeder:
    """Hands the samples to a live pipeline in order: `chunk` rows per push_imu call (None: all that are due in one call)."""

    def __init__(self, pl, imu, chunk=None):
        self.pl, self.imu, self.chunk, self.cur = pl, imu, chunk, 0

    def to(self, end):
        end = min(end, len(self.imu))
        while self.cur < end:
            k = end if self.chunk is None else min(end, self.cur + self.chunk)
            self.pl.push_imu(self.imu[self.cur:k])
            self.cur = k

    def upto(self, t):
        """The samples up to time t and the first one past it."""
        self.to(int(np.searchsorted(self.imu[:, 0], t, side="right")) + 1)


def push_live(pl, feeder, frames, ts, how):
    """A push after each frame's chunk of samples, retried with one more sample while the ring does not cover it (where the
    reference's FirstThr waits)."""
    from rebvo_b200 import capi
    for t in ts:
        feeder.upto(t)
    while True:
        try:
            return push(pl, frames, ts, how)
        except capi.RbError as e:
            assert _code(e) == RB_ERR_STATE, str(e)
            assert feeder.cur < len(feeder.imu)
            feeder.to(feeder.cur + 1)


def _from(imu, t):
    """The samples after t: a ring a few frames deep cannot hold the quarter second the stream has before its first frame,
    which the first frame's window (0, t0] skips anyway."""
    return imu[imu[:, 0] > t]


def run_live(p, ts, fr, batch, imu, how="host", fmt="rgb", sample_time=None, buffer_size=None, chunk=None,
             up_front=True, pl=None):
    """(nav, odometry) of a live-mode run: the samples all up front (or as the pushes need them), `batch`-frame pushes.
    sample_time: dataset mode's step on these samples by default."""
    from rebvo_b200 import capi
    own = pl is None
    if own:
        pl = capi.Pipeline(p, max_batch=batch)
        pl.set_odometry(True)
        pl.set_imu_live(_imu_params(), _dataset_tsample(imu) if sample_time is None else sample_time,
                        buffer_size or len(imu) + 16)
    try:
        feeder = Feeder(pl, imu, chunk)
        if up_front:
            feeder.to(len(imu))
        navs, odos = [], []
        for s in range(0, len(ts), batch):
            src = fr[s:s + batch, ..., 0] if fmt == "mono" else fr[s:s + batch]
            navs.append(push_live(pl, feeder, src, ts[s:s + batch], how))
            odos.append(pl.odometry())
        return np.concatenate(navs), np.concatenate(odos)
    finally:
        if own:
            pl.close()


def run_dataset(p, ts, fr, batch, imu, how="host", fmt="rgb"):
    r = run_pipeline(p, ts, fr, batch, how=how, fmt=fmt, imu=imu, odometry=True, collect=("odometry",))
    return r.nav, r.odometry


def assert_same(a, b, what):
    (nav_a, odo_a), (nav_b, odo_b) = a, b
    assert len(nav_a) == len(nav_b), what
    diff = np.nonzero((raw(nav_a) != raw(nav_b)).reshape(len(nav_a), -1).any(1))[0]
    assert len(diff) == 0, "%s: nav records differ from frame %d" % (what, diff[0])
    assert raw(odo_a).tobytes() == raw(odo_b).tobytes(), "%s: odometry records" % what


@pytest.mark.parametrize("how", ["host", "dev"])
@pytest.mark.parametrize("fmt", ["rgb", "mono"])
@pytest.mark.parametrize("batch", [1, 7, 10])
def test_live_up_front_is_dataset_mode(built, stream, batch, fmt, how):
    p, ts, fr, imu = stream
    want = run_dataset(p, ts, fr, batch, imu, how, fmt)
    assert np.isfinite(want[0]["Pos"]).all() and want[1]["tracked"][1:].all()
    assert_same(run_live(p, ts, fr, batch, imu, how, fmt), want, "live, all samples up front (%d, %s, %s)" % (batch, fmt, how))


@pytest.mark.parametrize("feed", ["one_at_a_time", "frame_chunks", "small_ring"])
def test_live_incremental_is_dataset_mode(built, stream, feed):
    p, ts, fr, imu = stream
    batch, kw = {"one_at_a_time": (7, dict(chunk=1)), "frame_chunks": (10, dict()),
                 "small_ring": (1, dict(buffer_size=35))}[feed]
    want = run_dataset(p, ts, fr, batch, imu)
    got = run_live(p, ts, fr, batch, _from(imu, -0.02), sample_time=_dataset_tsample(imu), up_front=False, **kw)
    assert_same(got, want, "live, samples fed %s" % feed)


def test_uncovered_push_changes_nothing(built, stream):
    """A push whose last frames the ring does not cover fails before it enqueues anything: the last push's records stay,
    and after the missing samples the run continues as an uninterrupted one."""
    from rebvo_b200 import capi
    p, ts, fr, imu = stream
    batch = 5
    want = run_dataset(p, ts, fr, batch, imu)
    pl = capi.Pipeline(p, max_batch=batch)
    try:
        pl.set_odometry(True)
        pl.set_imu_live(_imu_params(), _dataset_tsample(imu), 64)
        feeder = Feeder(pl, _from(imu, -0.02))
        navs, odos = [], []
        for s in range(0, NF, batch):
            if s == 10:   # frames 10..14 with samples up to frame 12 only
                feeder.upto(ts[12])
                before = pl.odometry()
                _raises(RB_ERR_STATE, pl.push, fr[s:s + batch], ts[s:s + batch])
                assert raw(pl.odometry()).tobytes() == raw(before).tobytes()
                assert len(pl.map(0).keylines()) == navs[-1][-1]["kn"]   # the newest map is still frame 9's
            navs.append(push_live(pl, feeder, fr[s:s + batch], ts[s:s + batch], "host"))
            odos.append(pl.odometry())
    finally:
        pl.close()
    assert_same((np.concatenate(navs), np.concatenate(odos)), want, "after an uncovered push")


def test_overflowing_push_imu_stores_nothing(built, stream):
    from rebvo_b200 import capi
    p, ts, fr, imu = stream
    want = run_dataset(p, ts, fr, 1, imu)
    pl = capi.Pipeline(p, max_batch=1)
    try:
        pl.set_odometry(True)
        pl.set_imu_live(_imu_params(), _dataset_tsample(imu), 30)
        feeder = Feeder(pl, _from(imu, -0.02))
        navs, odos = [], []
        for i in range(NF):
            if i == 8:   # four frames ahead do not fit in 30 samples: refused whole
                ahead = int(np.searchsorted(feeder.imu[:, 0], ts[11], side="right")) + 1
                _raises(RB_ERR_STATE, pl.push_imu, feeder.imu[feeder.cur:ahead])
            navs.append(push_live(pl, feeder, fr[i:i + 1], ts[i:i + 1], "host"))
            odos.append(pl.odometry())
    finally:
        pl.close()
    assert_same((np.concatenate(navs), np.concatenate(odos)), want, "after an overflowing push_imu")


def _unreleased(imu, t):
    """Index of the first sample a frame window ending at t leaves in the ring (the 1e-12 rule of SeachByTimeStamp)."""
    j = int(np.searchsorted(imu[:, 0], t, side="left"))
    return j + 1 if j < len(imu) and imu[j, 0] - t < 1e-12 else j


def test_reset_keeps_the_ring(built, stream):
    """rb_pipeline_reset in live mode starts the filter over and keeps the samples the ring has not released, with its read
    position.  Against the same pipeline history whose ring is replaced, at the reset, by a new one that holds exactly those
    samples.  (In IMU mode a reset pipeline does not give a new pipeline's records, so both runs share the history.)"""
    from rebvo_b200 import capi
    p, ts, fr, imu = stream
    batch, k = 5, 15
    st = _dataset_tsample(imu)
    out = []
    for refill in (False, True):
        pl = capi.Pipeline(p, max_batch=batch)
        try:
            pl.set_odometry(True)
            pl.set_imu_live(_imu_params(), st, len(imu) + 16)
            run_live(p, ts[:k], fr[:k], batch, imu, pl=pl)
            if refill:
                pl.set_imu_live(_imu_params(), st, len(imu) + 16)
                pl.push_imu(imu[_unreleased(imu, ts[k - 1]):])
            pl.reset()
            out.append(run_live(p, ts[k:], fr[k:], batch, imu[:0], pl=pl, up_front=False))
        finally:
            pl.close()
    assert_same(out[0], out[1], "live mode after reset")


def test_switching_modes(built, stream):
    """set_imu and set_imu_live replace each other: the mode set last is the one that runs, on top of the pipeline's history."""
    from rebvo_b200 import capi
    p, ts, fr, imu = stream
    batch, k = 10, 10
    st = _dataset_tsample(imu)
    live = run_live(p, ts, fr, batch, imu)
    navs = []
    for first in ("live", "dataset"):
        pl = capi.Pipeline(p, max_batch=batch)
        try:
            pl.set_odometry(True)
            if first == "live":
                pl.set_imu(imu, _imu_params())
                pl.set_imu_live(_imu_params(), st, len(imu) + 16)
                assert_same(run_live(p, ts, fr, batch, imu, pl=pl), live, "dataset mode replaced by live mode")
            else:
                pl.set_imu_live(_imu_params(), st, len(imu) + 16)
                pl.push_imu(imu[:40])
                pl.set_imu(imu, _imu_params())
                for s in range(0, NF, batch):
                    pl.push(fr[s:s + batch], ts[s:s + batch])
            # then dataset mode and a reset, in both pipelines
            pl.set_imu(imu, _imu_params())
            pl.reset()
            _raises(RB_ERR_ARG, pl.push_imu, imu[:1])   # dataset mode takes no samples
            navs.append(pl.push(fr[k:k + batch], ts[k:k + batch]))
        finally:
            pl.close()
    assert raw(navs[0]).tobytes() == raw(navs[1]).tobytes()


def test_argument_and_state_errors(built, stream):
    from rebvo_b200 import capi
    p, ts, fr, imu = stream
    pl = capi.Pipeline(p, max_batch=2)
    try:
        _raises(RB_ERR_ARG, pl.push_imu, imu[:3])   # IMU mode off
        for st, bs in ((0.0, 10), (-0.005, 10), (float("nan"), 10), (0.005, 0), (0.005, -3)):
            _raises(RB_ERR_ARG, pl.set_imu_live, _imu_params(), st, bs)
        pl.set_imu_live(_imu_params(), 0.005, 20)
        _raises(RB_ERR_ARG, pl.push_imu, imu[[3, 2]])                  # backwards within a call
        pl.push_imu(imu[5:8])
        _raises(RB_ERR_ARG, pl.push_imu, imu[6:7])                     # older than the last one stored
        pl.push_imu(imu[7:8])                                          # (equal is in order)
        _raises(RB_ERR_STATE, pl.push_imu, imu[8:25])                  # 17 do not fit beside 4: none stored
        pl.push_imu(imu[8:24])                                         # 16 do
        _raises(RB_ERR_STATE, pl.push_imu, imu[24:25])
        _raises(RB_ERR_STATE, pl.push, fr[:2], np.array([1.0, 1.05]))  # no sample at or past t = 1.0
        _raises(RB_ERR_ARG, pl.set_mirror, 1)                          # not in IMU mode, as in dataset mode
        _raises(RB_ERR_ARG, pl.set_depth, capi.depth_params())
    finally:
        pl.close()


def test_live_mode_vs_reference(built, tmp_path):
    """The pipeline in live mode against the reference's REBVO in ImuMode=1 (SampleTime 0.005, CircBufferSize 1000), the
    samples pushed frame by frame by oracle/ref_live_imu.cpp; and the same driver on the shim."""
    from oracle import ref_live_imu, refapi
    from rebvo_b200 import capi, synth
    if not (os.path.exists(ref_live_imu.EXE) and os.path.exists(ref_live_imu.SHIM_EXE)):
        pytest.skip("oracle/_ref/ref_live_imu / shim_live_imu not built (need the reference sources)")
    n_frames = 50
    seq = euroc_sequence()
    ts, fr = seq.frames(n_frames)
    imu = synth.imu_samples(seq, n_frames)
    p = capi.default_params(synth.EUROC)
    kv = refapi.ref_params_from(p, InitBias=1, InitBiasFrameNum=5)
    path = frames_file(tmp_path, ts, fr)
    _, ref = ref_live_imu.run(path, imu, str(tmp_path / "ref.bin"), kv)
    _, shim = ref_live_imu.run(path, imu, str(tmp_path / "shim.bin"), kv, exe=ref_live_imu.SHIM_EXE)
    nav, _ = run_live(p, ts, fr, 10, imu, sample_time=0.005, buffer_size=1000, up_front=False)
    n = min(len(ref), len(nav))
    print("live IMU mode: K ref %.12g gpu %.12g shim %.12g" % (ref["K"][n - 1], nav["K"][n - 1], shim["K"][-1]))
    assert np.isfinite(nav["Pos"][:n]).all()
    assert_knife_edge(ref, nav, n_frames - 2, "live IMU pipeline")
    assert np.allclose(ref["K"][1:n], nav["K"][1:n], rtol=1e-6, atol=1e-12)   # (record 0 is the untracked first frame)
    m = min(len(ref), len(shim))
    assert_knife_edge(ref, shim, n_frames - 2, "live IMU shim")
    assert np.allclose(ref["K"][:m], shim["K"][:m], rtol=1e-6, atol=1e-12)
