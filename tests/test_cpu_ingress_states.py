"""The ingress states of tests/ingress_states.py on the CPU: the NumPy restatement of the undistortion map equals the
reference's image_undistort bit for bit, every map case reaches what it is built for, and the pipeline cases of
tests/test_gpu_ingress.py cover every instance of rb_gray_enqueue's dispatch and every batch shape they are meant to, so
that a failure on the device points at a kernel, not at a case that missed its target."""
import numpy as np
import pytest

import ingress_states as S


def _need_ref():
    from oracle import refapi
    if not refapi.available():
        pytest.skip("oracle/_ref not built")


@pytest.mark.parametrize("name", sorted(S.MAPS))
def test_map_restatement_equals_reference(name):
    """undistort_map + apply_map (integer biInterp) == the reference's undistort_rgb on random and edge frames."""
    _need_ref()
    c = S.MAPS[name]
    m = S.map_of(name)
    for key in (("rand", 0), ("rand", 1), ("edge", 2)):
        rgb = S.frame(c["cam"], key)
        ref = S.ref_undistort(c["cam"], c["kc"], rgb)
        got = S.apply_map(m, rgb)
        assert np.array_equal(ref, got), (name, key, int((ref != got).sum()))


@pytest.mark.parametrize("name", sorted(S.MAPS))
def test_map_reach(name):
    c = S.MAPS[name]
    r = S.reach(S.map_of(name), c["cam"])
    print(name, r)
    for k, want in c["reach"].items():
        assert r[k] >= want, (name, k, r[k], want)
    # the valid taps are the product of the valid columns {floor, floor + 1} and rows: 0, 1, 2 or 4, never 3
    assert r["taps3"] == 0
    # every map: the two runs of a pair at every byte phase of its first tap, RGB (3 ix mod 4) and mono (ix mod 4, phase 3
    # taking the second word)
    for k in range(4):
        assert r["rgb_phase%d" % k] >= 1000 and r["mono_phase%d" % k] >= 1000, (name, k)


def test_map_reach_together():
    """What no single map has to reach, the maps together do: every tap count but 3, both paths, the last row pair and
    ug_pixel's last_word clamp, taps at pixel 0 and N - 1, ppx / ppy on integers and on x.5, exact (1, 0, 0, 0) weights."""
    tot = {}
    for name, c in S.MAPS.items():
        for k, v in S.reach(S.map_of(name), c["cam"]).items():
            tot[k] = tot.get(k, 0) + v
    for k in ("taps0", "taps1", "taps2", "taps4", "pair", "nonpair", "last_rows", "rgb_clamp", "tap0", "tapN",
              "zero_weight", "exact_one"):
        assert tot[k] >= 1, k
    pps = [(c["cam"]["ppx"] % 1, c["cam"]["ppy"] % 1) for c in S.MAPS.values()]
    assert (0.0, 0.0) in pps and (0.5, 0.5) in pps
    sizes = {(c["cam"]["w"], c["cam"]["h"]) for c in S.MAPS.values()}
    assert sizes >= {(752, 480), (1241, 376), (1226, 370), (1239, 375), (640, 480), (1280, 960)}


def test_white_frame_integral_exceeds_float_mantissa():
    """The all-255 1280x960 frame's integral ends at 765 N > 2^24: the order of every pass's additions shows in the planes."""
    cam = S.CAMS["1280x960"]
    g = S.frame(cam, ("white",)).astype(np.int64).sum(2)
    assert g.sum() == 765 * cam["w"] * cam["h"] and g.sum() > 2 ** 24


def test_cases_cover_every_instance_and_shape():
    """The GPU cases run all 18 instances of k_gray<MONO, L> / k_undistort_gray<IMGS, MONO, L>, batch sizes 1-3, 4, 5, 7, 8
    (IMGS = 4 with tails 0, 1, 3), 31 and 64, in 64-frame workspaces and in workspaces of exactly the batch's size, every
    placement, and both box plans at m = 1, 2, 5, 64 on each of the four scale-space geometries."""
    assert len(S.INSTANCES) == 18
    got = set()
    for c in S.CASES:
        got |= S.case_instances(c)
    assert got == S.INSTANCES, sorted(S.INSTANCES - got, key=str)
    batches = {(nb, c["B"]) for c in S.CASES for n in c["sizes"] for nb in S.sub_batches(c, n)}
    ms = {nb for nb, _ in batches}
    assert ms >= {1, 2, 3, 4, 5, 7, 8, 31, 64}
    assert any(b == 64 and nb < 64 for nb, b in batches) and any(b == nb for nb, b in batches)
    # device RGB at every byte offset on a w % 4 == 0 camera without undistortion (k_gray<false, GRAY_ALIGNED>)
    offs = {o for c in S.CASES if c["how"] == "dev" and c["m"] == "rgb" and c["und"] is None
            and S.CAMS[c["cam"]]["w"] % 4 == 0 for o in c["offsets"]}
    assert offs == {0, 1, 2, 3}
    assert any(c["imu"] for c in S.CASES)
    # the rest of a head / rest push at an odd byte of the staging: an odd head on 1239x375 (N odd), RGB and mono
    odd = [c for c in S.CASES if c["how"] == "host" and c["cam"] == "1239x375" and (c["sub"] or 8) % 2 == 1
           and any(len(S.sub_batches(c, n)) == 2 for n in c["sizes"])]
    assert {c["m"] for c in odd} == {"rgb", "mono"}
    for cam in ("752x480", "1241x376", "1239x375", "1280x960"):
        for s in S.SIGMAS:
            c = [c for c in S.CASES if c["id"] == "sspace_%s_s%.2f" % (cam, s)]
            assert len(c) == 1 and c[0]["B"] == 64 and set(c[0]["sizes"]) == {1, 2, 5, 64}
            assert S.case_keys(c[0], 8, 64)[-1] == ("white",)
