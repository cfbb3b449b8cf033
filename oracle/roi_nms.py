"""Seeded RoI-head-shaped inputs of `multiclass_nms` (test infrastructure): 1000 RoIs of a 640 x 640 image, 80 classes + background,
class-specific boxes (n, 4 * 80) clipped to the image, as the RoI head's get_bboxes passes them.  Shared by
oracle/make_golden_multiclass_nms_roi.py (which stores the reference's outputs in tests/golden/multiclass_nms_roi.npz) and the tests
that read that file; numpy's PCG64 stream makes the inputs the same everywhere, and the fixture stores their checksums.

Cases (score_thr 0.05, IoU 0.5):
  below       about 8 000 candidates: mmcv's offset branch (one NMS over all offset boxes)
  above       about 16 000 candidates: the split branch (class by class, then the merge)
  slow        `below` plus one RoI whose class-79 box lies in the negative corner and overlaps, after the class offset, the class-78
              box of a RoI at the far corner: the class offset does not separate the classes and the two branches differ
  factors     `below` with score_factors (the NMS ranks by score * factor)
  sparse      about 800 candidates, max_num=-1
  clustered   about 16 000 candidates on 8 objects (heavy overlap: few survivors), max_num=-1
"""
import numpy as np

N, C, SIDE = 1000, 80, 640.0
SCORE_THR, IOU = 0.05, 0.5
CASES = dict(below=dict(frac=0.1, seed=101, max_num=100),
             above=dict(frac=0.2, seed=102, max_num=100),
             slow=dict(frac=0.1, seed=103, max_num=100, planted=True),
             factors=dict(frac=0.1, seed=104, max_num=100, factors=True),
             sparse=dict(frac=0.01, seed=105, max_num=-1),
             clustered=dict(frac=0.2, seed=106, max_num=-1, clusters=8))


def inputs(name):
    """-> bboxes (N, 4C) fp32, scores (N, C+1) fp32, score_factors (N,) fp32 or None."""
    c = CASES[name]
    rng = np.random.default_rng(c['seed'])
    if c.get('clusters'):
        obj = rng.random((c['clusters'], 2)) * (SIDE - 80) + 40
        ctr = obj[rng.integers(0, c['clusters'], N)] + rng.normal(0, 2.0, (N, 2))
        wh = np.full((N, 2), 40.0) + rng.normal(0, 2.0, (N, 2))
    else:
        ctr = rng.random((N, 2)) * SIDE
        wh = rng.random((N, 2)) * 56 + 8
    base = np.concatenate([ctr - wh / 2, ctr + wh / 2], 1)
    boxes = np.clip(base[:, None, :] + rng.normal(0, 2.0, (N, C, 4)), 0, SIDE)
    x1, y1 = np.minimum(boxes[..., 0], boxes[..., 2]), np.minimum(boxes[..., 1], boxes[..., 3])
    x2, y2 = np.maximum(boxes[..., 0], boxes[..., 2]), np.maximum(boxes[..., 1], boxes[..., 3])
    boxes = np.stack([x1, y1, x2, y2], -1)
    hit = rng.random((N, C)) < c['frac']
    scores = np.where(hit, 0.05 + 0.9 * rng.random((N, C)), 0.05 * rng.random((N, C)))
    scores = np.concatenate([scores, rng.random((N, 1))], 1)
    if c.get('planted'):
        boxes[0] = [-30, -30, -2, -2]                       # class 79 of RoI 0: the negative corner
        boxes[1] = [615, 615, 640, 640]                     # class 78 of RoI 1: the far corner, IoU 0.69 after the offset
        scores[0, :C], scores[1, :C] = 0, 0
        scores[0, C - 1], scores[1, C - 2] = 0.99, 0.98
    factors = rng.random(N).astype(np.float32) if c.get('factors') else None
    return boxes.reshape(N, 4 * C).astype(np.float32), scores.astype(np.float32), factors


def checksum(a):
    return np.float64(np.asarray(a, dtype=np.float64).sum())
