"""All of the pipeline's optional per-frame outputs at once (keyline mirror, odometry records, depth grid and dense depth
image) across a host push cut into two sub-batches: every output equals, byte for byte, the same run with that output
alone, with captured batches and with eager launches."""
import numpy as np
import pytest

import pipeline_util as pu
from test_gpu_depth_image import run_image

pytestmark = pytest.mark.gpu


def record_bytes(recs):
    """Mirror records as bytes: 15-byte net_keyline records whole, KeyLine records field by field (the four bytes between
    c_p and rho are the struct's padding and hold no value)."""
    if recs.dtype == np.uint8:
        return recs.tobytes()
    return b"".join(np.ascontiguousarray(recs[k]).tobytes() for k in recs.dtype.names)


@pytest.mark.parametrize("graph", [True, False], ids=["graph", "eager"])
@pytest.mark.parametrize("mirror", [1, 2])
def test_all_outputs_equal_each_alone(built, monkeypatch, mirror, graph):
    from rebvo_b200 import capi, synth
    # 12-frame host pushes: a 2-frame head, then 10 frames whose copy runs beside it (REBVO_B200_SUB=2)
    monkeypatch.setenv("REBVO_B200_SUB", "2")
    if not graph:
        monkeypatch.setenv("REBVO_B200_NO_GRAPH", "1")
    ts, fr = pu.euroc_stream(24, seed=13)
    prm = capi.default_params(synth.EUROC)

    def run(**kw):
        out = dict(mirror=0, mode=0, depth=False, odometry=False)
        out.update(kw)
        return run_image(prm, ts, fr, 12, **out)

    every = run(mirror=mirror, mode=2, depth=True, odometry=True)
    alone = {"mirror": run(mirror=mirror), "odometry": run(odometry=True), "grid": run(depth=True),
             "image": run(depth=True, mode=2)}
    what = "mirror %d, %s" % (mirror, "graph" if graph else "eager")
    for k, r in alone.items():
        assert pu.raw(every["nav"]).tobytes() == pu.raw(r["nav"]).tobytes(), "%s: nav records against %s alone" % (what, k)
    assert len(every["mirrors"]) == len(alone["mirror"]["mirrors"]) == 24
    for f, (a, b) in enumerate(zip(every["mirrors"], alone["mirror"]["mirrors"])):
        assert record_bytes(a) == record_bytes(b), "%s: mirror records of frame %d" % (what, f)
    assert pu.raw(every["odometry"]).tobytes() == pu.raw(alone["odometry"]["odometry"]).tobytes(), what
    assert len(every["grids"]) == len(alone["grid"]["grids"]) == 24
    for f, ((ca, ma), (cb, mb)) in enumerate(zip(every["grids"], alone["grid"]["grids"])):
        assert ca.tobytes() == cb.tobytes() and np.float64(ma).tobytes() == np.float64(mb).tobytes(), (
            "%s: grid of frame %d" % (what, f))
    assert len(every["images"]) == len(alone["image"]["images"]) == 24
    for f, (a, b) in enumerate(zip(every["images"], alone["image"]["images"])):
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes(), "%s: image of frame %d" % (what, f)
