"""The front-end states of tests/front_states.py on the CPU: each state reaches what it is built for, and the NumPy
restatement (plane_fit.port_detect, port_reestimate, port_field) equals the unmodified reference on it bit for bit, so a
failure of the device comparison (tests/test_gpu_front_states.py) points at a kernel, not at a state that missed its
target."""
import numpy as np
import pytest

import front_states as fs
from parity_util import KL_EXACT_DETECT


def _need_ref():
    from oracle import refapi
    if not refapi.available():
        pytest.skip("oracle/_ref not built")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def same_detect(a, b, tag, skip_undefined=None):
    """Step results a and b (dicts of run_port / run_ref / run_dev) equal bit for bit.  skip_undefined: the restatement's
    step results, whose NaN reEstimateThresh values mark the reference's undefined read of a never-written kl[0]."""
    assert [a["kn"], a["t"], a["l"]] == [b["kn"], b["t"], b["l"]], (tag, a["kn"], b["kn"], a["t"], b["t"])
    assert len(a["kl"]) == len(b["kl"]), tag
    for f in KL_EXACT_DETECT:
        assert np.array_equal(_bits(a["kl"][f]), _bits(b["kl"][f])), (tag, f)
    assert np.array_equal(a["mask"], b["mask"]), (tag, "mask", int((a["mask"] != b["mask"]).sum()))
    for i, (x, y) in enumerate(zip(a["reest"], b["reest"])):
        if skip_undefined is not None and np.isnan(skip_undefined["reest"][i]):
            continue
        assert np.float32(x).view(np.uint32) == np.float32(y).view(np.uint32), (tag, "reest", i, x, y)


# minimum reach of all states of one window size together
TOTAL_WANT = dict(p_id_collisions=500, clamp_max=6, clamp_min=6, err_pos=6, err_neg=6,
                  cut_lane0=1, cut_lane31=1, cut_thread_first=1, cut_thread_last=1, cut_last_chunk=2,
                  **{"q%d_p%d" % (a, b): 1 for a in range(4) for b in range(4)})


@pytest.mark.parametrize("R", [1, 2, 3, 4])
def test_detect_states(R, tmp_path):
    _need_ref()
    jobs = fs.detect_jobs(R)
    refs = fs.ref_results(tmp_path, R, jobs)
    total = {}
    for job, ref in zip(jobs, refs):
        port = fs.run_port(job)
        for s, (p, r) in enumerate(zip(port, ref)):
            same_detect(p, r, "%s step %d" % (job["name"], s), skip_undefined=p)
        c = fs.reach(job, port)
        print(job["name"], "kn", [r["kn"] for r in port][:6], {k: v for k, v in c.items() if v})
        for k, v in job["want"].items():
            assert c.get(k, 0) >= v, (job["name"], k, c.get(k, 0), v)
        for k, v in c.items():
            total[k] = total.get(k, 0) + v
    print("R=%d total" % R, total)
    if R <= 2:   # the wider windows' sums leave a last-bit residue on the axis-aligned edges
        assert total.get("tx_zero", 0) + total.get("ty_zero", 0) >= 4 and total.get("neg_zero", 0) >= 4, total
    for k, v in TOTAL_WANT.items():
        assert total.get(k, 0) >= v, (R, k, total.get(k, 0), v)


def _ref_map(cam):
    from oracle import refapi
    return refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], fs.SIGMA0, fs.KSIGMA)


def test_reestimate_states():
    """reEstimateThresh on loaded keylines: knum <= 0, 1, kn - 1, kn, > kn; 1, 2, 100 and 4096 bins; kn = 1, a zero range,
    two values, bins hit exactly, 50 000 keylines mostly in one bin."""
    _need_ref()
    cam = fs.CAM
    mask = np.full((cam["h"], cam["w"]), -1, np.int32)
    exact = 0
    for name, n_m in fs.reest_sets():
        m = _ref_map(cam)
        kl = fs.keylines_with(n_m)
        m.set_keylines(kl)
        m.set_mask(mask, len(kl))
        for k, n in fs.reest_calls(len(kl)):
            want = np.float32(m.reestimate(k, n)[1])
            got = fs.port_reestimate(n_m, k, n)
            assert want.view(np.uint32) == got.view(np.uint32), (name, k, n, want, got)
        if name.startswith("exact_bins"):
            mx, mn = n_m.max(), n_m.min()
            q = np.float32(len(n_m) - 1) * (mx - n_m) / (mx - mn)
            exact += int((q == np.round(q)).sum())
    print("keylines on an exact bin edge:", exact)
    assert exact >= 4000


def test_field_states():
    """build_field on loaded keyline sets: winner id on every pixel and its distance where there is one."""
    _need_ref()
    cam = fs.CAM
    w, h = cam["w"], cam["h"]
    mask = np.full((h, w), -1, np.int32)
    for name, kl, runs, min_ties in fs.field_sets(w, h, 3000):
        m = _ref_map(cam)
        m.set_keylines(kl)
        m.set_mask(mask, len(kl))
        ties = 0
        for radius, min_mod in runs:
            m.build_field(radius, min_mod)
            want = m.field()
            got = fs.port_field(kl, radius, min_mod, w, h)
            assert np.array_equal(want[:, :, 1], got[:, :, 1]), (name, radius, min_mod)
            won = want[:, :, 1] >= 0
            assert np.array_equal(want[:, :, 0][won], got[:, :, 0][won]), (name, radius, min_mod)
            ties += fs.field_ties(kl, radius, min_mod, w, h) if len(kl) <= 3000 else 0
        print(name, "kn", len(kl), "ties", ties)
        assert ties >= min_ties, (name, ties)
