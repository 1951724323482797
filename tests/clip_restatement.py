"""TEST INFRASTRUCTURE — CPU restatement of the clip volumes (DESIGN.md §9.15), independent of simlod_b200, on top of
query_restatement's point predicate and pick_restatement's frame.

  keep_mask(clip, samples)                             per sample: whether the clip draws it
  clipped_pick(clip, records, samples, u, w, h)        the (h, w) int64 frame of indices of the clipped frame

`clip` is anything with the fields of SimlodClip (mode, num_regions, regions). The clipped frame is pick_frame over the
view export with the clipped samples taken out of the candidates and the indices of the others kept: a clipped sample's
position is replaced by NaN, which pick_frame's projection never places inside the frame."""
import numpy as np

import pick_restatement as P
import query_restatement as Q

NONE, INSIDE, OUTSIDE = 0, 1, 2


def keep_mask(clip, samples):
    """NONE: every sample. Else `in` = the region query's predicate holds for one of the first num_regions regions;
    INSIDE keeps what is in, OUTSIDE what is not."""
    n = len(samples)
    if clip is None or clip.mode == NONE:
        return np.ones(n, dtype=bool)
    if clip.mode not in (INSIDE, OUTSIDE):
        raise ValueError("unknown clip mode %r" % clip.mode)
    inside = np.zeros(n, dtype=bool)
    for k in range(clip.num_regions):
        inside |= Q.contains(clip.regions[k], samples)
    return inside if clip.mode == INSIDE else ~inside


def clipped_pick(clip, records, samples, u, width, height):
    s = np.array(samples, copy=True)
    drop = ~keep_mask(clip, s)
    for c in ("x", "y", "z"):
        s[c][drop] = np.nan
    return P.pick_frame(records, s, u, width, height)
