"""numpy restatement of qdtrack's BDD100K MOTS bitmask (external/qdtrack/qdtrack/core/to_bdd100k/utils.py:15-38): mask_prepare reads
each instance of a frame's track_result dict in dict order, mask_merge paints them in np.argsort order of their scores with the
reference's own channel arithmetic.  pycocotools.mask.decode is unicorn_b200.results.rle_decode (column-major runs), and the bitmask
has the frame's own size instead of the hard-coded SHAPE = [720, 1280].  The tests compare the device painter (unicorn_b200.bdd) with
this, and tools/bench_bdd_bitmask.py times it as the host baseline."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from unicorn_b200.results import rle_decode  # noqa: E402


def decode(segm):
    """pycocotools.mask.decode of one RLE dict: uint8 [h, w]."""
    counts = segm["counts"]
    h, w = (int(v) for v in segm["size"])
    return rle_decode(counts.decode("ascii") if isinstance(counts, bytes) else counts, h, w).astype(np.uint8)


def mask_prepare(track_dict):
    """utils.py:15-22."""
    scores, colors, masks = [], [], []
    for id_, instance in track_dict.items():
        masks.append(decode(instance["segm"]))
        colors.append([instance["label"] + 1, 0, id_ >> 8, id_ & 255])
        scores.append(instance["bbox"][-1])
    return scores, colors, masks


def mask_merge(mask_infor, h, w):
    """utils.py:24-38 up to the PNG: the uint8 [h, w, 4] array PIL saves."""
    scores, colors, masks = mask_infor
    bitmask = np.zeros((h, w, 4), dtype=np.uint8)
    sorted_idxs = np.argsort(scores)
    for idx in sorted_idxs:
        for i in range(4):
            bitmask[..., i] = bitmask[..., i] * (1 - masks[idx]) + masks[idx] * colors[idx][i]
    return bitmask


def bdd_bitmask(track_dict, h, w):
    """The seg_track bitmask of one frame of size h x w from its track_result dict."""
    return mask_merge(mask_prepare(track_dict), h, w)
