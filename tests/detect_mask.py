"""Detection masks in the NumPy detector restatement: plane_fit.port_detect with build_mask's candidate test gated by a
w x h byte mask, where a zero byte at (x, y) keeps pixel (x, y) from being a candidate (rb_map_detect_masked,
rb_pipeline_set_detect_mask, rb_pipeline_push_masked).  Everything after the candidate test -- the raster-order
compaction, the kl_max cut, join_edges and the threshold feedback -- is port_detect's own."""
import numpy as np

import plane_fit


def port_detect_masked(img0, dog, R, pos_neg, dog_thresh, kl_max, tresh, l_kl_num, kl_ref, gain, tmax, tmin, ppx, ppy,
                       keep=None, mask=None):
    """port_detect (same arguments and results) with the candidates restricted to the pixels where keep != 0; keep = None
    is port_detect itself."""
    args = (img0, dog, R, pos_neg, dog_thresh, kl_max, tresh, l_kl_num, kl_ref, gain, tmax, tmin, ppx, ppy, mask)
    if keep is None:
        return plane_fit.port_detect(*args)
    keep = np.asarray(keep)
    terms = plane_fit.detect_terms

    def gated(img0_, dog_, R_):
        T = terms(img0_, dog_, R_)
        # -inf fails the gradient test (n2gI < t1 * t1) at every threshold: a masked pixel is not a candidate
        T["n2gI"] = np.where(keep[T["ys"], T["xs"]] != 0, T["n2gI"], np.float32(-np.inf)).astype(np.float32)
        return T

    plane_fit.detect_terms = gated
    try:
        return plane_fit.port_detect(*args)
    finally:
        plane_fit.detect_terms = terms


def candidates(img0, dog, R, pos_neg, dog_thresh, tresh):
    """Flat pixel indices of build_mask's candidates in raster order (before any mask and cut) at the threshold used."""
    T = plane_fit.detect_terms(img0, dog, R)
    P = plane_fit.detect_tests(T, R, pos_neg, dog_thresh, tresh)
    ok = P["grad"] & P["pn"] & P["sub"] & P["dog"]
    return (T["ys"][ok] * dog.shape[1] + T["xs"][ok]).astype(np.int64)


def mask_families(w, h, R, cand, kl_max, seed=0):
    """{name: uint8 [h, w]} masks that reach what the masked detector must get right: none and every pixel masked, a
    50 % random mask, a rectangle, single zero bytes on chosen candidates, masks that move the kl_max cut (the first
    candidates masked, and every candidate after the cut masked), and the R-margin alone zeroed (no interior pixel
    changes)."""
    rng = np.random.default_rng(seed)
    out = {"ones": np.ones((h, w), np.uint8), "zeros": np.zeros((h, w), np.uint8),
           "random": (rng.random((h, w)) < 0.5).astype(np.uint8) * rng.integers(1, 256, (h, w), dtype=np.uint8)}
    rect = np.ones((h, w), np.uint8)
    rect[h // 4:h // 2, w // 3:2 * w // 3] = 0
    out["rect"] = rect
    single = np.ones((h, w), np.uint8).reshape(-1)
    if len(cand):
        single[cand[rng.choice(len(cand), min(len(cand), 12), replace=False)]] = 0
        single[cand[0]] = single[cand[-1]] = 0
    out["single"] = single.reshape(h, w)
    first = np.ones((h, w), np.uint8).reshape(-1)
    first[cand[:max(1, kl_max // 2)]] = 0                 # the cut moves to a later candidate
    out["cut_later"] = first.reshape(h, w)
    after = np.ones((h, w), np.uint8).reshape(-1)
    after[cand[kl_max:]] = 0                              # exactly kl_max candidates are left: the same cut
    out["cut_same"] = after.reshape(h, w)
    margin = np.ones((h, w), np.uint8)
    margin[:R] = margin[-R:] = 0
    margin[:, :R] = margin[:, -R:] = 0
    out["margin"] = margin
    return out
