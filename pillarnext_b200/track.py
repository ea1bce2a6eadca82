"""Velocity-based greedy tracking of the detector's output, per sequence and class: CenterPoint's tracker (Yin et al.,
CVPR 2021, "Center-based 3D Object Detection and Tracking"), restated here because its code is not part of the
reference.  It is the consumer of the CenterHead's velocity output (`vel`).

  * Order.  A frame belongs to a sequence (the Waymo context name) and has a timestamp in microseconds.  The frames of
    a sequence run in ascending timestamp; dt = (t_k - t_{k-1}) * 1e-6 s (the exact integer difference, times 1e-6 in
    fp64, rounded to fp32; 0 for a sequence's first frame).  Classes are tracked independently.
  * Frame.  A detection's BEV centre (x, y) and velocity (vx, vy) go into the global frame through the frame's 4x4
    pose (sensor -> global): p_x = ((T00 x + T01 y) + T02 z) + T03, v_x = T00 vx + T01 vy (likewise for y), in fp64
    from the fp32 box, no fused multiply-add, then rounded to fp32 once.  Association uses global positions only; the
    returned boxes are unchanged.
  * Association, per frame, for each detection with score >= min_score: its back-projected position b = p - v dt
    (fp32, each product rounded, no fused multiply-add), and its distance to live track j, d = sqrt(dx^2 + dy^2) with
    (dx, dy) = b - q_j (fp32, in that order).  A pair is valid when d <= max_dist[class].  Detections are visited in
    descending score, ties by lower index; each takes the valid, still unclaimed track with the smallest d, ties to
    the older track (lower id), and a detection that finds none starts a new track.  Tracks born in this frame are not
    candidates in it.
  * Update, after all detections of the frame: a matched track takes q <- p, v <- the detection's v, misses <- 0; an
    unmatched one coasts, q <- q + v dt (fp32), misses += 1, and is dropped when misses > max_age.  A dropped object
    seen again starts a new track.
  * Ids: consecutive integers per sequence, from 0, in order of birth (frame, then class index, then visit order).
    Detections below min_score get tracking id -1 and neither start nor continue a track.
  * Defaults: max_dist vehicle 2.0 m, pedestrian 1.0 m, cyclist 1.5 m (MAX_DIST, Waymo's classes at 10 Hz).  A class
    outside that table needs an entry in max_dist.  NUSCENES_MAX_DIST holds the entries for nuScenes' tracking classes
    at its 2 Hz key frames, where the velocity back-projection spans 0.5 s: car 4.0 m, truck 4.0 m, bus 5.0 m, trailer
    3.0 m, motorcycle 4.0 m, bicycle 2.5 m, pedestrian 1.0 m; evaluate_nuscenes_tracking.track_and_score passes them.
    All of these are this project's choice, not values taken from CenterPoint's released tracker.

At most 4096 tracks (pnx_track_max_tracks()) of one (sequence, class) may be live at once, counting those born in the
current frame; more raise ValueError.  The tracker runs on the GPU (pnx_track_greedy, csrc/track.cu: one warp per
(sequence, class), the tracks in shared memory); `host=True` runs its host twin, which equals it bit for bit.
oracle/track_oracle.py restates the same definition sequentially in numpy."""
import numpy as np
import torch

MAX_DIST = {"vehicle": 2.0, "pedestrian": 1.0, "cyclist": 1.5}
NUSCENES_MAX_DIST = {"car": 4.0, "truck": 4.0, "bus": 5.0, "trailer": 3.0, "motorcycle": 4.0, "bicycle": 2.5,
                     "pedestrian": 1.0}


def split_token(token):
    """Waymo token "<context_name>-<timestamp_micros>" -> (context_name, timestamp), as the reference's evaluation()
    splits it."""
    parts = str(token).split("-")
    return parts[0], int(parts[1])


def class_max_dist(class_names, max_dist=None):
    table = dict(MAX_DIST, **(max_dist or {}))
    missing = [n for n in class_names if n not in table]
    if missing:
        raise ValueError("no max_dist for classes %s: pass max_dist={name: metres}" % missing)
    return np.array([table[n] for n in class_names], np.float32)


def frame_order(frames):
    """tokens ordered by (sequence, timestamp), the sequences and each sequence's first frame (seq_start [S + 1])."""
    tokens = sorted(frames, key=lambda t: (str(frames[t]["sequence"]), int(frames[t]["timestamp"])))
    seqs, seq_start = [], []
    for i, t in enumerate(tokens):
        s = str(frames[t]["sequence"])
        if not seqs or seqs[-1] != s:
            seqs.append(s)
            seq_start.append(i)
        elif int(frames[t]["timestamp"]) == int(frames[tokens[i - 1]]["timestamp"]):
            raise ValueError("sequence %s: two frames at timestamp %d" % (s, int(frames[t]["timestamp"])))
    return tokens, seqs, np.array(seq_start + [len(tokens)], np.int32)


def _arr(x, dtype):
    return (x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)).astype(dtype, copy=False)


def pack(detections, frames, class_names, max_dist=None):
    """The flat arrays pnx_track_greedy takes (numpy): frames in (sequence, timestamp) order, detections concatenated
    frame by frame in index order, and the 64-bit sort keys (segment f C + c, then descending score)."""
    unknown = sorted(set(detections) - set(frames))
    if unknown:
        raise ValueError("detections for tokens without a frame: %s" % unknown[:5])
    tokens, seqs, seq_start = frame_order(frames)
    C = len(class_names)
    boxes, scores, seg, count = [np.zeros((0, 9), np.float32)], [np.zeros(0, np.float32)], [np.zeros(0, np.int64)], []
    for f, t in enumerate(tokens):
        d = detections.get(t)
        n = 0
        if d is not None:
            b = _arr(d["box3d_lidar"], np.float32).reshape(-1, 9)
            s = _arr(d["scores"], np.float32).reshape(-1)
            lab = _arr(d["label_preds"], np.int64).reshape(-1)
            if not (len(b) == len(s) == len(lab)):
                raise ValueError("frame %s: box3d_lidar, scores and label_preds differ in length" % t)
            if len(lab) and (lab.min() < 0 or lab.max() >= C):
                raise ValueError("frame %s: label_preds outside [0, %d)" % (t, C))
            if np.isnan(s).any():
                raise ValueError("frame %s: NaN scores" % t)
            boxes.append(b)
            scores.append(s + np.float32(0.0))                 # -0 -> +0: equal scores order by index
            seg.append(f * C + lab)
            n = len(b)
        count.append(n)
    boxes, scores, seg = np.concatenate(boxes), np.concatenate(scores), np.concatenate(seg)
    u = scores.view(np.uint32).astype(np.int64)
    ordered = np.where(scores >= 0, u | 0x80000000, (~u) & 0xFFFFFFFF)
    seg_count = np.bincount(seg, minlength=len(tokens) * C).astype(np.int32)
    poses = np.stack([np.asarray(frames[t]["pose"], np.float64).reshape(4, 4) for t in tokens]) if tokens else \
        np.zeros((0, 4, 4))
    return dict(tokens=tokens, sequences=seqs, seq_start=seq_start, frame_count=np.array(count, np.int64),
                boxes=boxes, scores=scores, keys=(seg << 32) | (0xFFFFFFFF - ordered),
                seg_start=(np.cumsum(seg_count) - seg_count).astype(np.int32), seg_count=seg_count, poses=poses,
                times=np.array([int(frames[t]["timestamp"]) for t in tokens], np.int64),
                max_dist=class_max_dist(class_names, max_dist))


def run_device(pk, max_age, min_score):
    """track_id [D] (numpy int64) of a pack() on the GPU: one key sort, the tracker, one copy back."""
    from . import ops
    dev = torch.device("cuda", torch.cuda.current_device())

    def cu(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    order = torch.sort(cu(pk["keys"]), stable=True)[1]
    return ops.track_greedy(cu(pk["boxes"]), cu(pk["scores"]), order, cu(pk["seg_start"]), cu(pk["seg_count"]),
                            cu(pk["poses"]), cu(pk["times"]), cu(pk["seq_start"]), cu(pk["max_dist"]), max_age,
                            min_score).cpu().numpy()


def run_host(pk, max_age, min_score):
    """The same through the host twin (pnx_track_greedy_host)."""
    from . import ops
    order = np.argsort(pk["keys"], kind="stable").astype(np.int64)
    return ops.track_greedy_host(pk["boxes"], pk["scores"], order, pk["seg_start"], pk["seg_count"], pk["poses"],
                                 pk["times"], pk["seq_start"], pk["max_dist"], max_age, min_score)


def track(detections, frames, class_names, max_dist=None, max_age=3, min_score=0.0, host=False):
    """detections: token -> {"box3d_lidar" [K, 9], "scores" [K], "label_preds" [K]} (predict's output; tensors or
    arrays), labels indexing class_names; frames: token -> {"sequence", "timestamp" (int microseconds), "pose" [4, 4]
    sensor -> global}.  max_dist: {class name: metres} overriding the defaults.  Returns token -> the detection's dict
    plus "tracking_id" [K] int64 (a CPU tensor, or a numpy array when the scores are not a tensor), for every token of
    `detections`."""
    if int(max_age) < 0:
        raise ValueError("max_age must be >= 0, got %r" % (max_age,))
    pk = pack(detections, frames, class_names, max_dist)
    ids = (run_host if host else run_device)(pk, int(max_age), float(min_score))
    out, at = {}, np.cumsum(np.concatenate([[0], pk["frame_count"]]))
    for f, t in enumerate(pk["tokens"]):
        if t not in detections:
            continue
        tid = ids[at[f]:at[f + 1]].copy()
        d = dict(detections[t])
        d["tracking_id"] = torch.from_numpy(tid) if torch.is_tensor(d["scores"]) else tid
        out[t] = d
    return out
