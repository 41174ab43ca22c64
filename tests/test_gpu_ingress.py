"""The front of the frame against the reference, plane by plane: the gray pass, the fused undistortion and the batched scale
space of the pipeline, read back with Pipeline.batch_plane after each push and compared bit for bit (as uint32) with the
reference's undistort_rgb -> rgb2bw -> sspace::build planes of the same frame.  The cases (tests/ingress_states.py) run every
instance of k_gray<MONO, L> and k_undistort_gray<IMGS, MONO, L>, batch sizes 1 to 64 in workspaces larger than the batch and
of its size, host pushes as the head and as the rest sub-batch, device buffers at byte offsets 0..3 (RGB24; mono8 aligned),
strided host and device frames, graph replays with a new source each time, and one IMU-mode push."""
import numpy as np
import pytest

import ingress_states as S

pytestmark = pytest.mark.gpu

# row steps of strided frame i, from the tight one (as test_gpu_frames.py's "mixed")
STEPS = (lambda r: r, lambda r: r + 1, lambda r: r + 3, lambda r: r + 61, lambda r: -(-r // 512) * 512)


def _place(frames, mem):
    """Each frame in a buffer of its own, at byte offset i % 4, rows STEPS[i % 5] bytes apart, 0xa5 around and between the
    rows: NumPy views (mem "host") or torch CUDA views (mem "dev")."""
    import torch
    n, h, w = frames.shape[:3]
    bpp = 3 if frames.ndim == 4 else 1
    out = []
    for i in range(n):
        s, off = STEPS[i % 5](w * bpp), i % 4
        buf = np.full(off + h * s + 5, 0xa5, np.uint8)
        buf[off:off + h * s].reshape(h, s)[:, :w * bpp] = frames[i].reshape(h, w * bpp)
        shape, strides = ((h, w, 3), (s, 3, 1)) if bpp == 3 else ((h, w), (s, 1))
        if mem == "host":
            out.append(np.lib.stride_tricks.as_strided(buf[off:], shape, strides))
        else:
            out.append(torch.from_numpy(buf).cuda()[off:].as_strided(shape, strides))
    return out


def _push(pl, case, k, fr, ts):
    mono = case["m"] == "mono"
    how = case["how"]
    if how == "host":
        return pl.push_mono(fr, ts) if mono else pl.push(fr, ts)
    if how in ("shost", "sdev"):
        return pl.push_frames(_place(fr, "host" if how == "shost" else "dev"), ts)
    import torch
    off = case["offsets"][k % len(case["offsets"])]
    flat = np.ascontiguousarray(fr).reshape(-1)
    buf = torch.full((flat.size + off + 8,), 0xa5, dtype=torch.uint8, device="cuda")
    buf[off:off + flat.size] = torch.from_numpy(flat).cuda()
    torch.cuda.synchronize()
    try:
        return (pl.push_mono_dev if mono else pl.push_dev)(buf.data_ptr() + off, ts)
    finally:
        del buf


def _bits_equal(a, b):
    return np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("case", S.CASES, ids=[c["id"] for c in S.CASES])
def test_batch_planes_bitwise(built, case, monkeypatch):
    from oracle import refapi
    from rebvo_b200 import capi, synth
    if not refapi.available():
        pytest.skip("oracle/_ref not built")
    if case["sub"]:
        monkeypatch.setenv("REBVO_B200_SUB", str(case["sub"]))
    else:
        monkeypatch.delenv("REBVO_B200_SUB", raising=False)
    cam, kc = S.case_cam(case), S.case_kc(case)
    total = sum(case["sizes"])
    ts = np.arange(total) / 20.0
    pl = capi.Pipeline(capi.default_params(cam, Sigma0=case["sigma"]), max_batch=case["B"])
    try:
        with pytest.raises(capi.RbError):   # no batch yet
            pl.batch_plane(0, "gray")
        if kc is not None:
            pl.set_undistort(kc)
        if case["imu"]:
            seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=11, zf=cam["zfx"])
            pl.set_imu(synth.imu_samples(seq, total), capi.default_imu_params(InitBias=1, InitBiasFrameNum=5))
        first = 0
        for k, n in enumerate(case["sizes"]):
            keys = S.case_keys(case, first, n)
            _push(pl, case, k, S.frames(cam, keys, mono=case["m"] == "mono"), ts[first:first + n])
            m = S.sub_batches(case, n)[-1]   # the slots hold the last sub-batch: the rest of a head / rest push
            with pytest.raises(capi.RbError):
                pl.batch_plane(m, "gray")
            for slot in range(m):
                exp = S.expected(cam, kc, case["sigma"], keys[n - m + slot])
                for p in ("gray", "img0", "dog"):
                    got = pl.batch_plane(slot, p)
                    assert _bits_equal(got, exp[p]), "%s push %d (%d frames) slot %d/%d plane %s: %d pixels differ" % (
                        case["id"], k, n, slot, m, p, int((got.view(np.uint32) != exp[p].view(np.uint32)).sum()))
            first += n
    finally:
        pl.close()
