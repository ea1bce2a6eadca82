"""Sequential restatement of pillarnext_b200.evaluate_nuscenes_tracking.nuscenes_tracking_metrics (TEST INFRASTRUCTURE
-- see oracle/__init__.py), independent of the product.

One (scene, class, cutoff) at a time, frames in order: the pairs by nds_oracle.center_distance's fp64 arithmetic on
the fp32 centres, the carry-over in pair order, then waymo_hungarian_oracle.assign (scipy's linear_sum_assignment plus
the tie rule) on the cardinality-first weights 2^40 - round(d 2^26) of the remaining pairs.  Fragmentations are found
by a different route than the product's: a per-object "missed since its last match" flag set in every frame where the
object has a box and no match.

`defects` switches on one deliberate error each, for the tests that show a comparison can fail: "no_carry_over",
"not_cardinality_first" (the weight 2^27 + 1 - round(d 2^26), which can prefer one close pair to two far ones),
"threshold_off_by_one" (the cutoff at the (n_k + 1)-th match) and "no_frag"."""
import math

import numpy as np

from oracle import gts_oracle
from oracle.nds_oracle import CLASS_RANGE, _box9, _np, center_distance
from oracle.waymo_hungarian_oracle import assign

F32 = np.float32
TRACKING_NAMES = ("bicycle", "bus", "car", "motorcycle", "pedestrian", "trailer", "truck")
RECALLS = np.linspace(0.1, 1.0, 40)
DEFECTS = ("no_carry_over", "not_cardinality_first", "threshold_off_by_one", "no_frag")


def _weight(d, defects):
    dq = int(math.floor(float(d) * 2.0 ** 26 + 0.5))
    return float((2 ** 27 + 1 if "not_cardinality_first" in defects else 2 ** 40) - dq)


def load(gts, tracks, class_names, class_range=None):
    """-> (tracking classes, frames): per frame in (scene, timestamp) order, (scene, boxes [(name, box9, id)] left by
    the filters, detections [(score, index, name, box9, tracking id)] of the tracking classes with id >= 0)."""
    from det3d.datasets.pipelines.sample_ops import libm_trig
    tcls = [n for n in class_names if n in TRACKING_NAMES]
    ranges = dict(CLASS_RANGE, **(class_range or {}))
    tokens = sorted(gts, key=lambda t: (str(gts[t]["sequence"]), int(gts[t]["timestamp"])))
    frames = []
    for t in tokens:
        g = gts[t]
        boxes = [_box9(b) for b in _np(g["boxes"]).reshape(len(g["names"]), -1)]
        if "num_points" in g:
            counts = [int(n) for n in _np(g["num_points"])]
        else:
            b9 = np.array(boxes, np.float32).reshape(-1, 9)
            pts = np.asarray(_np(g["points"]), np.float32)[:, :3]
            counts = list(gts_oracle.points_in_boxes(pts, b9, libm_trig(b9[:, 8])).sum(0)) if len(boxes) else []
        kept = [(n, b, str(i)) for n, b, i, k in zip(g["names"], boxes, g["ids"], counts)
                if n in tcls and math.sqrt(b[0] * b[0] + b[1] * b[1]) < ranges[n] and k > 0]
        dets = []
        d = tracks.get(t)
        if d is not None:
            db, ds, dl, di = _np(d["box3d_lidar"]), _np(d["scores"]), _np(d["label_preds"]), _np(d["tracking_id"])
            mine = [i for i in range(len(ds)) if class_names[int(dl[i])] in tcls and int(di[i]) >= 0]
            if len(mine) > 500:
                raise ValueError("more than 500 detections in frame %r" % t)
            for i in mine:
                name, box = class_names[int(dl[i])], _box9(db[i])
                if math.sqrt(box[0] * box[0] + box[1] * box[1]) < ranges[name]:
                    dets.append((F32(ds[i]) + F32(0.0), i, name, box, int(di[i])))
        frames.append((str(g["sequence"]), kept, dets))
    return tcls, frames


def run(frames, name, cut, defects=()):
    """One class at cutoff `cut` (None: every detection) -> (tp, fp, fn, ids, frag, sum d, matched {(frame, det)})."""
    tp = fp = fn = ids = frag = 0
    dsum = 0.0
    matched = set()
    last, missed = {}, {}                                   # object -> last matched id; object -> missed since then
    for f, (scene, boxes, dets) in enumerate(frames):
        gi = [j for j, b in enumerate(boxes) if b[0] == name]
        live = sorted([d for d in dets if d[2] == name and (cut is None or d[0] >= cut)], key=lambda d: (-d[0], d[1]))
        dist = {}
        for d in live:
            for j in gi:
                v = center_distance(d[3], boxes[j][1])
                if v < 2.0:
                    dist[(d[1], j)] = F32(v)
        tid = {d[1]: d[4] for d in live}
        obj = lambda j: (scene, boxes[j][2])                 # noqa: E731
        kept = {}
        if "no_carry_over" not in defects:
            for d in live:
                for j in sorted(j for (i, j) in dist if i == d[1]):
                    if d[1] in kept or j in kept.values():
                        continue
                    if last.get(obj(j)) == d[4]:
                        kept[d[1]] = j
        w = {p: _weight(v, defects) for p, v in dist.items() if p[0] not in kept and p[1] not in kept.values()}
        m = assign(w, [d[1] for d in live if d[1] not in kept])
        pairs = list(kept.items()) + list(m.items())
        for i, j in pairs:
            o = obj(j)
            ids += o in last and last[o] != tid[i]
            frag += missed.get(o, False) and "no_frag" not in defects
            last[o], missed[o] = tid[i], False
            dsum += float(dist[(i, j)])
            matched.add((f, i))
        hit = {j for _, j in pairs}
        for j in gi:
            if j not in hit and obj(j) in last:
                missed[obj(j)] = True
        tp += len(pairs)
        fp += len(live) - len(pairs)
        fn += len(gi) - len(pairs)
    return tp, fp, fn, ids, frag, dsum, matched


def class_cutoffs(frames, name, defects=()):
    """The reached recalls' cutoffs in recall order, and P."""
    P = sum(1 for _, boxes, _ in frames for b in boxes if b[0] == name)
    *_, matched = run(frames, name, None, defects)
    ms = sorted((d[0] for f, (_, _, dets) in enumerate(frames) for d in dets if (f, d[1]) in matched), reverse=True)
    cuts = []
    for r in RECALLS:
        n = int(np.ceil(r * P)) + ("threshold_off_by_one" in defects)
        if P == 0 or n > len(ms):
            break
        cuts.append(ms[n - 1])
    return cuts, P


def tracking_metrics(gts, tracks, class_names, class_range=None, defects=()):
    """Same inputs and outputs as nuscenes_tracking_metrics (plus `defects`, see the module docstring)."""
    tcls, frames = load(gts, tracks, class_names, class_range)
    nan = float("nan")
    per_class = {}
    for name in tcls:
        cuts, P = class_cutoffs(frames, name, defects)
        res = {"n_gt": P}
        if P == 0:
            res.update({k: nan for k in ("AMOTA", "AMOTP", "MOTA", "MOTP", "recall", "IDS", "FRAG", "FP", "FN",
                                         "score_cutoff")})
        elif not cuts:
            res.update(AMOTA=0.0, AMOTP=2.0, MOTA=0.0, MOTP=nan, recall=0.0, IDS=0, FRAG=0, FP=0, FN=P, score_cutoff=nan)
        else:
            amota, amotp, best = 0.0, 2.0 * (len(RECALLS) - len(cuts)), None
            for k, cut in enumerate(cuts):
                tp, fp, fn, ids, frag, dsum, _ = run(frames, name, cut, defects)
                r = RECALLS[k]
                amota += max(0.0, 1.0 - (ids + fp + fn - (1.0 - r) * P) / (r * P))
                motp = dsum / tp if tp else 2.0
                amotp += motp
                mota = max(0.0, 1.0 - (fn + fp + ids) / P)
                if best is None or mota > best[0]:
                    best = (mota, motp, tp / P, ids, frag, fp, fn, float(cut))
            res.update(AMOTA=amota / len(RECALLS), AMOTP=amotp / len(RECALLS),
                       **dict(zip(("MOTA", "MOTP", "recall", "IDS", "FRAG", "FP", "FN", "score_cutoff"), best)))
        per_class[name] = res
    out = {}
    scored = [v for v in per_class.values() if v["n_gt"] > 0]
    for key in ("AMOTA", "AMOTP", "MOTA", "MOTP", "recall"):
        vals = [v[key] for v in scored if not math.isnan(v[key])]
        out[key] = float(np.mean(vals)) if vals else nan
    for key in ("IDS", "FRAG", "FP", "FN"):
        out[key] = int(sum(v[key] for v in scored)) if scored else nan
    out["per_class"] = per_class
    return out
