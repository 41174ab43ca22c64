"""Mono8 input (rb_pipeline_push_mono / _dev, rb_map_upload_mono).  A mono frame m is defined to be the RGB24 frame
(m, m, m), so every result must equal the RGB path's on the replicated frames bit for bit: the gray plane, the keylines
and masks, the nav records (compared as raw bytes), the host mirror, and the IMU-mode records.  The synthetic streams
are gray replicated into three channels, so the mono frames are their first channel."""
import numpy as np
import pytest

from pipeline_util import EUROC_KC, assert_runs_identical, euroc_sequence, keylines_equal, push, raw, run_pipeline, \
    run_reference

pytestmark = pytest.mark.gpu

NF = 40


@pytest.fixture(scope="module")
def stream():
    seq = euroc_sequence()
    ts, rgb = seq.frames(NF)
    assert np.array_equal(rgb[..., 0], rgb[..., 1]) and np.array_equal(rgb[..., 0], rgb[..., 2])
    return seq, ts, rgb, np.ascontiguousarray(rgb[..., 0])


def _stream_run(stream, fmt, batch, how="host", kc=None, mirror=0, imu=False, n=NF):
    """the first n frames of the stream in `batch`-frame pushes (fmt: 'rgb', 'mono' or one of them per push), with the
    two newest maps after the last push and every frame's mirror records"""
    from rebvo_b200 import capi, synth
    seq, ts, rgb, _ = stream
    return run_pipeline(capi.default_params(synth.EUROC), ts[:n], rgb[:n], batch, how, fmt, kc=kc, mirror=mirror,
                        imu=synth.imu_samples(seq, n) if imu else None,
                        collect=("maps", "mirrors") if mirror else ("maps",))


def _ramp_frame(w, h):
    """every value 0..255 (the first row counts up), blocks of random levels and 255 / 0 plateaus"""
    rng = np.random.default_rng(11)
    img = np.kron(rng.integers(0, 256, (h // 16 + 1, w // 16 + 1)), np.ones((16, 16), np.int64))[:h, :w]
    img[: h // 4, w // 2:] = 255
    img[h // 2: h // 2 + 40, 100:300] = 255
    img[-60:, -120:] = 0
    img[0] = np.arange(w) % 256
    img[1] = 255 - np.arange(w) % 256
    assert set(np.unique(img)) == set(range(256))
    return img.astype(np.uint8)


@pytest.mark.parametrize("which", ["stream", "ramp"])
def test_stage_gray_and_detect(built, stream, which):
    """rb_map_upload_mono vs rb_map_upload_rgb of the replicated frame: the gray plane, then the keylines and the id mask
    after the scale space and the detector."""
    from rebvo_b200 import capi, synth
    cam = synth.EUROC
    mono = stream[3][5] if which == "stream" else _ramp_frame(cam["w"], cam["h"])
    rgb = np.repeat(mono[:, :, None], 3, axis=2)
    p = capi.default_params(cam)
    ctx = capi.Ctx(cam, p.Sigma0, p.KSigma, kl_capacity=40000)
    got = []
    for upload, img in (("upload_rgb", rgb), ("upload_mono", mono)):
        m = ctx.new_map()
        getattr(m, upload)(img)
        gray = m.plane("gray")
        m.dog_build()
        kn, t, l = m.detect(p.det, p.DetectorThresh, 0)
        got.append((gray, kn, t, l, m.keylines(), m.mask(), m.plane("dog")))
        m.close()
    ctx.close()
    (g0, kn0, t0, l0, kl0, mk0, d0), (g1, kn1, t1, l1, kl1, mk1, d1) = got
    assert np.array_equal(g0.view(np.uint32), g1.view(np.uint32))
    assert np.array_equal(g1, 3.0 * mono.astype(np.float32))
    assert np.array_equal(d0.view(np.uint32), d1.view(np.uint32))
    assert kn0 == kn1 and kn1 > 100 and (t0, l0) == (t1, l1)
    assert keylines_equal(kl0, kl1)
    assert np.array_equal(mk0, mk1)


@pytest.mark.parametrize("kc", [None, EUROC_KC], ids=["plain", "undistort"])
@pytest.mark.parametrize("how", ["host", "device"])
def test_pipeline_mono_equals_rgb(built, stream, monkeypatch, kc, how):
    """Byte-identical nav records and equal newest maps for batch sizes 20, 7 and 1, and with host pushes cut into a
    5-frame head and the rest (REBVO_B200_SUB=5)."""
    for batch in (20, 7, 1):
        assert_runs_identical(_stream_run(stream, "rgb", batch, how, kc), _stream_run(stream, "mono", batch, how, kc),
                              "batch %d" % batch)
    monkeypatch.setenv("REBVO_B200_SUB", "5")
    assert_runs_identical(_stream_run(stream, "rgb", 20, how, kc), _stream_run(stream, "mono", 20, how, kc), "SUB=5")


def test_graph_replay_equals_eager_mono(built, stream, monkeypatch):
    a = _stream_run(stream, "mono", 10, kc=EUROC_KC)
    monkeypatch.setenv("REBVO_B200_NO_GRAPH", "1")
    b = _stream_run(stream, "mono", 10, kc=EUROC_KC)
    assert_runs_identical(a, b, "eager")
    assert_runs_identical(_stream_run(stream, "rgb", 10, kc=EUROC_KC), b, "eager vs RGB")


@pytest.mark.parametrize("kc", [None, EUROC_KC], ids=["plain", "undistort"])
def test_alternating_formats(built, stream, kc):
    """One pipeline fed mono, RGB, mono, ... (the captured batches are kept per input format): the records of an all-RGB
    run, from host and from device memory."""
    ref = _stream_run(stream, "rgb", 5, kc=kc)
    assert_runs_identical(ref, _stream_run(stream, ["mono", "rgb"], 5, kc=kc), "mono/rgb")
    assert_runs_identical(ref, _stream_run(stream, ["rgb", "mono", "mono"], 5, "device", kc=kc),
                          "rgb/mono/mono, device")


@pytest.mark.parametrize("mode", [1, 2])
def test_mirror_mono(built, stream, mode):
    assert_runs_identical(_stream_run(stream, "rgb", 20, kc=EUROC_KC, mirror=mode),
                          _stream_run(stream, "mono", 20, kc=EUROC_KC, mirror=mode), "mirror %d" % mode)


@pytest.mark.parametrize("how", ["host", "device"])
def test_imu_mode_mono(built, stream, how):
    """IMU mode (the EuRoC mono + IMU configuration, with undistortion)."""
    a = _stream_run(stream, "rgb", 10, how, kc=EUROC_KC, imu=True)
    b = _stream_run(stream, "mono", 10, how, kc=EUROC_KC, imu=True)
    assert_runs_identical(a, b, "IMU mode")
    assert np.isfinite(a.nav["Pos"]).all()


def test_mono_vs_reference(built, stream, tmp_path):
    """The mono push against the unmodified reference run on the RGB frames, with the bars of the RGB trajectory test."""
    _, ts, rgb, _ = stream
    _, rec = run_reference(tmp_path, ts, rgb)
    nav = _stream_run(stream, "mono", 20).nav
    n = min(len(rec), NF - 1)
    assert n >= NF - 2
    assert np.array_equal(rec["kn"][:n], nav["kn"][:n])
    assert np.array_equal(rec["matches"][1:n], nav["matches"][1:n])
    d = rec["Pos"][:n] - nav["Pos"][:n]
    assert float(np.sqrt((d ** 2).sum(1).mean())) <= 1e-7
    assert np.abs(rec["PoseLie"][:n] - nav["PoseLie"][:n]).max() <= 1e-7
    assert np.allclose(rec["Kp"][1:n], nav["Kp"][1:n], rtol=1e-9, atol=0)
    assert np.array_equal(rec["est_ok"][1:n] != 0, nav["estimation_ok"][1:n] != 0)


def _bad_calls(pl, dev, mono, ts, B):
    import ctypes as C
    from rebvo_b200 import capi
    base = dev.data_ptr()
    assert base % 4 == 0
    nav = np.zeros(B + 1, capi.NAV)
    tsa = np.ascontiguousarray(ts[:B + 1])
    L, h = pl.L, pl.h_
    return [
        lambda: pl.push_mono(0, ts[:B]),                                                        # NULL frames
        lambda: pl.push_mono_dev(0, ts[:B]),
        lambda: pl.check(L.rb_pipeline_push_mono(h, capi._p(mono[:B]), None, B, capi._p(nav))),   # NULL ts
        lambda: pl.check(L.rb_pipeline_push_mono_dev(h, C.c_void_p(base), None, B, capi._p(nav))),
        lambda: pl.push_mono(mono[:0], ts[:0]),                                                 # n < 1
        lambda: pl.push_mono_dev(base, ts[:0]),
        lambda: pl.check(L.rb_pipeline_push_mono(h, capi._p(mono[:B]), capi._p(tsa), -1, capi._p(nav))),
        lambda: pl.push_mono(mono[:B + 1], tsa),                                                # n > max_batch
        lambda: pl.push_mono_dev(base, tsa),
        lambda: pl.push_mono_dev(base + 1, ts[:B]),                                             # misaligned
        lambda: pl.push_mono_dev(base + 2, ts[:B]),
        lambda: pl.push_mono_dev(base + 3, ts[:B]),
    ]


def test_bad_arguments(built, stream):
    """NULL frames or timestamps, n < 1, n > max_batch and a misaligned device pointer raise, before and between valid
    pushes; the valid pushes give the records of a pipeline that never saw the bad calls."""
    import torch
    from rebvo_b200 import capi, synth
    _, ts, _, mono = stream
    B, n = 5, 15
    ref = _stream_run(stream, "mono", B, n=n).nav
    pl = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=B)
    dev = torch.from_numpy(np.ascontiguousarray(mono[:n])).cuda()
    navs = []
    for s in range(0, n, B):
        for call in _bad_calls(pl, dev, mono, ts, B):
            with pytest.raises(capi.RbError):
                call()
        navs.append(push(pl, mono[s:s + B], ts[s:s + B]))
    pl.close()
    del dev
    assert np.array_equal(raw(np.concatenate(navs)), raw(ref))


def test_bench_pass_mono(built, stream):
    """Measurement hook: pass 6 (mono -> gray) and 7 (undistortion + mono -> gray) with their algorithmic bytes."""
    from rebvo_b200 import capi, synth
    _, ts, _, mono = stream
    pl = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=8)
    push(pl, mono[:8], ts[:8])
    N = synth.EUROC["w"] * synth.EUROC["h"]
    ms, by = pl.bench_pass(6, 8, 3)
    assert ms > 0 and by == 5.0 * N * 8
    with pytest.raises(capi.RbError):   # pass 7 needs the undistortion map
        pl.bench_pass(7, 8, 3)
    pl.set_undistort(EUROC_KC)
    for nimg in (8, 3):
        ms, by = pl.bench_pass(7, nimg, 3)
        assert ms > 0 and by == 5.0 * N * nimg + 32.0 * N
    pl.close()
