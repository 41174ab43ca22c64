"""The per-frame map chain after the minimiser: k_match (FordwardMatch's apply + directed_matching against the unrotated
old map) and k_reg_ekf (gate + Regularize_1_iter + EKF + rotate_keylines of the old map), against the four-kernel chain
k_fm_apply_rotate -> k_directed_match -> k_regularize_a_gate -> k_regb_ekf (REBVO_B200_MAP_CHAIN=0).  Both must give the
same bits: raw nav records, the keylines and masks of the two newest maps, and per frame the FordwardMatch winners,
directed hits and regularised keylines."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NF = 72
EUROC_KC = (-0.28340811, 0.07395907, 0.0, 0.00019359, 1.76187114e-05)   # GlobalConfig_EuRoC_2.txt, UseUndistort=1


@pytest.fixture(scope="module")
def stream():
    from rebvo_b200 import synth
    cam = synth.EUROC
    ts, rgb = synth.Sequence(w=cam["w"], h=cam["h"], seed=7, zf=cam["zfx"]).frames(NF)
    return ts, rgb


@pytest.fixture(scope="module")
def special(stream):
    """the stream with a black first frame (frame 1 tracks against an empty old map), a black frame 30 (nothing to
    track: the NaN guard clears do_match) and frame 45 taken from another scene (few matches: the mapping gate closes)"""
    from rebvo_b200 import synth
    cam = synth.EUROC
    ts, rgb = stream
    rgb = rgb.copy()
    rgb[0] = 0
    rgb[30] = 0
    rgb[45] = synth.Sequence(w=cam["w"], h=cam["h"], seed=99, zf=cam["zfx"]).frames(1)[1][0]
    return ts, rgb


def _raw(nav):
    return np.ascontiguousarray(nav).view(np.uint8)


def _keylines_equal(a, b):
    from rebvo_b200 import capi
    if len(a) != len(b):
        return False
    return all(np.array_equal(a[f], b[f], equal_nan=True) for f in capi.KEYLINE.names)


def _run(frames, batch, how="host", kc=None, mirror=0):
    """nav records of the frames pushed in `batch`-frame pushes, the keylines + masks of the two newest maps after the
    last push, the mirror records per frame, and (batch 1) the newest map's counters after every push"""
    from rebvo_b200 import capi, synth
    ts, rgb = frames
    pl = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=batch)
    if kc is not None:
        pl.set_undistort(kc)
    if mirror:
        pl.set_mirror(mirror)
    navs, mirrors, counters = [], [], []
    for s in range(0, len(ts), batch):
        if how == "host":
            nav = pl.push(rgb[s:s + batch], ts[s:s + batch])
        else:
            import torch
            dev = torch.from_numpy(np.ascontiguousarray(rgb[s:s + batch])).cuda()
            nav = pl.push_dev(dev.data_ptr(), ts[s:s + batch])
            del dev
        navs.append(nav)
        for i in range(len(nav) if mirror else 0):
            mirrors.append(pl.mirror(i).copy())
        if batch == 1:
            counters.append(pl.map(0).counters())
    maps = []
    for age in (0, 1):
        m = pl.map(age)
        maps.append((m.keylines(), m.mask()))
    pl.close()
    return np.concatenate(navs), maps, mirrors, counters


def _both(monkeypatch, *args, **kw):
    """the run with the two-kernel chain (the default) and with REBVO_B200_MAP_CHAIN=0"""
    a = _run(*args, **kw)
    with monkeypatch.context() as m:
        m.setenv("REBVO_B200_MAP_CHAIN", "0")
        b = _run(*args, **kw)
    return a, b


def _assert_same(ab, what):
    (nav_a, maps_a, mir_a, cnt_a), (nav_b, maps_b, mir_b, cnt_b) = ab
    assert len(nav_a) == len(nav_b)
    diff = np.nonzero((_raw(nav_a) != _raw(nav_b)).reshape(len(nav_a), -1).any(1))[0]
    assert len(diff) == 0, "%s: nav records differ from frame %d" % (what, diff[0])
    for age in (0, 1):
        assert _keylines_equal(maps_a[age][0], maps_b[age][0]), "%s: keylines of map %d" % (what, age)
        assert np.array_equal(maps_a[age][1], maps_b[age][1]), "%s: mask of map %d" % (what, age)
    assert len(mir_a) == len(mir_b)
    for i, (x, y) in enumerate(zip(mir_a, mir_b)):
        ok = np.array_equal(x, y) if x.dtype == np.uint8 else _keylines_equal(x, y)
        assert ok, "%s: mirror records of frame %d" % (what, i)
    for i, (x, y) in enumerate(zip(cnt_a, cnt_b)):
        assert x == y, "%s: frame %d: (fwd_match, nmatch, reg_num) %r against %r" % (what, i, x, y)


@pytest.mark.parametrize("kc", [None, EUROC_KC], ids=["plain", "undistort"])
@pytest.mark.parametrize("how", ["host", "device"])
def test_chain_equals_four_kernel_chain(built, stream, monkeypatch, kc, how):
    for batch in (64, 7, 1):
        ab = _both(monkeypatch, stream, batch, how, kc)
        _assert_same(ab, "batch %d" % batch)
    nav, cnt = ab[0][0], ab[0][3]
    # both matchers and the regularisation did work on this stream
    assert (nav["fwd_matches"] > 0).sum() >= NF // 2 and (nav["matches"] > 0).sum() >= NF // 2
    assert sum(c[2] > 0 for c in cnt) >= NF // 2


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_chain_mirror(built, stream, monkeypatch, mode):
    """the host mirror of every frame's map (mode 1 keeps the rescaling inline on the tracker stream)"""
    _assert_same(_both(monkeypatch, stream, 20, kc=EUROC_KC, mirror=mode), "mirror %d" % mode)


@pytest.mark.parametrize("env", ["REBVO_B200_OVERLAP", "REBVO_B200_MIN_PERSIST", "REBVO_B200_NO_GRAPH"])
def test_chain_schedules(built, stream, monkeypatch, env):
    """one stream without the side streams (OVERLAP=0), the one-launch-per-evaluation minimiser whose arg-max is its
    own kernel (MIN_PERSIST=0), and eager launches (NO_GRAPH=1)"""
    monkeypatch.setenv(env, "1" if env == "REBVO_B200_NO_GRAPH" else "0")
    _assert_same(_both(monkeypatch, stream, 20), env)


def test_chain_special_frames(built, special, monkeypatch):
    """black frames, an empty old map and a frame whose match count closes the mapping gate"""
    from rebvo_b200 import capi, synth
    p = capi.default_params(synth.EUROC)
    for batch in (20, 1):
        ab = _both(monkeypatch, special, batch)
        _assert_same(ab, "batch %d" % batch)
    nav = ab[0][0]
    assert nav["kn"][0] == 0 and nav["kn"][30] == 0
    assert nav["kn"][1] > 0 and nav["matches"][1] < p.MatchThreshold   # tracked against the empty map of frame 0
    assert nav["estimation_ok"][30] == 0


def test_stage_profile_keys(built, stream, monkeypatch):
    """the eager stage profile runs the two-kernel chain and still reports every stage key as a number"""
    monkeypatch.setenv("REBVO_B200_STAGE_PROF", "1")
    from rebvo_b200 import capi, synth
    ts, rgb = stream
    res = []
    for chain in ("1", "0"):
        monkeypatch.setenv("REBVO_B200_MAP_CHAIN", chain)
        pl = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=16)
        nav = pl.push(rgb[:16], ts[:16])
        st, frames = pl.stage_profile()
        pl.close()
        assert frames == 16
        for k in ("minimizer", "quantile+field", "fwdmatch+rotate", "directed_match", "regularize+ekf", "rescale"):
            assert np.isfinite(st[k]) and st[k] >= 0, k
        assert st["quantile+field"] > 0 and st["directed_match"] > 0 and st["regularize+ekf"] > 0
        res.append(nav)
    assert np.array_equal(_raw(res[0]), _raw(res[1]))
