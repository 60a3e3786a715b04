"""TEST INFRASTRUCTURE ONLY -- the pose fits under occlusion of DESIGN.md section 24 restated in numpy, on top of the
unchanged oracles of the two fits.  An occluder mask O [H, W] (nonzero = something may be in front of the object)
leaves U = not O as the known pixels and the mask M' = M n U.

- The translation fit under O is translation_oracle.fit on a render whose O pixels read "no hit" (S' = S n U),
  against M'.
- The contour refinement under O is contour_refine_oracle.refine(..., occ=O): phi and the box size of M', and a
  contour pixel counted and paired only when it and its four neighbours lie in U.

`detection_occluders` restates nope_b200.crop.detection_occluders with a loop over the detections."""
import numpy as np

import contour_refine_oracle as cro
import translation_oracle as to


def hidden_render(render, occ):
    """the render callback with the O pixels read as "no hit" (depth 0)"""
    o = np.asarray(occ) != 0
    return lambda R, t: np.where(o, np.float32(0), np.asarray(render(R, t), dtype=np.float32))


# ------------------------------------------------------------------ translation
def fit_translation(render, R, t_init, mask, occ, K4, iters):
    """-> (t, iou, stats of S' at t) after `iters` updates of one hypothesis under O"""
    return to.fit(hidden_render(render, occ), R, t_init, cro.visible(mask, occ), K4, iters)


def translation_stats(D, mask, occ):
    """stats(S', M') of one render D [H, W] (0 = not hit)"""
    o = np.asarray(occ) != 0
    return to.stats((np.asarray(D) > 0) & ~o, cro.visible(mask, occ))


# ------------------------------------------------------------------ occluders from a frame's detections
def detection_occluders(masks, frame_idx):
    """uint8 [B, H, W]: the union of the other detections' masks of the same frame, minus the detection's own"""
    m = np.asarray(masks) != 0
    fi = np.asarray(frame_idx)
    out = np.zeros(m.shape, dtype=np.uint8)
    for b in range(len(m)):
        others = [j for j in range(len(m)) if j != b and fi[j] == fi[b]]
        if others:
            out[b] = m[others].any(0) & ~m[b]
    return out
