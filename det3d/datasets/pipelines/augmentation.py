"""Drop-in for the reference's global augmentation transforms (configs/dataset/preprocess/augmentation.yaml):
Rotation, Scaling, Translation and Flip, applied to a training frame in config order.

Import paths, constructor arguments and assertions are the reference's, and so are the random draws: the same
np.random calls in the same order (uniform for rotation and scaling, normal(0, noise, 1) for translation, one choice per
flip axis whose probability is > 0), so a seeded data-loader worker draws the reference's parameters.

Difference: __call__ does not transform res["points"] or the boxes.  It appends one record (code, p0, p1, p2) to
res["aug"]; scenes.collate packs the records into aug [B, 4, 4] float64, and the detector applies them on the GPU to the
points and raw boxes before label assignment (SingleStageDetector.global_aug, ops.global_aug, include/pnx.h).  Box
rotation, scaling, translation and flipping follow the reference's box_np_ops, NaN elements included."""
import numpy as np

# record codes of pnx_global_aug (include/pnx.h); 0 marks an empty slot
ROTATION, SCALING, TRANSLATION, FLIP = 1, 2, 3, 4


def _append(res, code, p0=0.0, p1=0.0, p2=0.0):
    res.setdefault("aug", []).append((float(code), float(p0), float(p1), float(p2)))
    return res


class Flip(object):
    """Mirror in y (x flip: y -> -y, yaw -> -yaw) and in x (y flip: x -> -x, yaw -> pi - yaw), each with its
    probability.  Record: (FLIP, fx, fy, 0)."""

    def __init__(self, flip_prob):
        self.flip_prob = flip_prob
        assert 0 <= flip_prob[0] < 1
        assert 0 <= flip_prob[1] < 1

    def _draw(self, p):
        if p <= 0:
            return False
        return bool(np.random.choice([False, True], replace=False, p=[1 - p, p]))

    def __call__(self, res):
        fx = self._draw(self.flip_prob[0])
        fy = self._draw(self.flip_prob[1])
        return _append(res, FLIP, fx, fy)


class Scaling(object):
    """Scale x, y, z (and box sizes and velocities) by s ~ U(scale).  Record: (SCALING, s, 0, 0)."""

    def __init__(self, scale):
        self.min_scale, self.max_scale = scale

    def __call__(self, res):
        return _append(res, SCALING, np.random.uniform(self.min_scale, self.max_scale))


class Rotation(object):
    """Rotate about z by theta ~ U(rotation).  Record: (ROTATION, theta, cos theta, sin theta), the cosine and sine
    taken by numpy here as the reference takes them."""

    def __init__(self, rotation):
        self.rotation = rotation

    def __call__(self, res):
        theta = np.random.uniform(self.rotation[0], self.rotation[1])
        return _append(res, ROTATION, theta, np.cos(theta), np.sin(theta))


class Translation(object):
    """Shift x, y and z by one t ~ N(0, noise).  Record: (TRANSLATION, t, 0, 0)."""

    def __init__(self, noise):
        self.noise = noise

    def __call__(self, res):
        t = np.random.normal(0, self.noise, 1)
        return _append(res, TRANSLATION, t[0])
