"""The training data path -- sweeps, ground-truth sampling, augmentation, label assignment -- chained by
SingleStageDetector.training_step at the reference experiments' production shapes, against the numpy oracles and the
host twins.

Recording.  oracle/reader_fixtures.py writes two info trees into tmp_path: nuScenes, 6 frames of 10 sweeps of 28k
points with 60 boxes each (a fifth of them with NaN velocity, sweep 1 stored without transform), and Waymo, 3 frames of
3 sweeps of 200k points with 150 boxes each, placed within +-36 m (a dense street).  The boxes are relabelled to a
street-like class mix -- nuScenes mostly cars, pedestrians, barriers and cones with one or none of each rarer class and
two names outside the class list; Waymo mostly vehicles with 2-12 pedestrians and 2-5 cyclists per frame -- so the
reference's sampler groups (nuScenes 2/3/7/4/6/2/6/6/2/2, Waymo 15/10/10) draw candidates in every frame, and the
sampler both accepts and rejects in every frame.  tools/create_gt_database.py cuts
the database on the GPU.  One batch of all frames is drawn through NuScenesDataset / WaymoDataset built from the
reference's composed experiment (tests/golden/ref_readers.npz) -- its sampler, global augmentation and label settings,
CBGS resampling and Waymo's drop_frames off so every sweep is there -- and collated by scenes.collate.  training_step
of the experiment's detector then runs with ops.accumulate_sweeps, gt_sample, global_aug and assign_labels wrapped
through pytest's MonkeyPatch (each call passes through unchanged; its device inputs and outputs are kept) and stops at
_forward, which is replaced by a stub that raises.  The library handle is a proxy that notes every pnx_* called.

What is compared, each stage on its own recorded inputs:
- sweeps: oracle/sweeps_oracle.accumulate and the host twin, bit for bit, tail rows and count included;
- sampling: oracle/gts_oracle.apply and the host twin, bit for bit: points (the rows past count are frame B and zeros),
  boxes, classes, accepted, count;
- augmentation: oracle/aug_oracle.apply and the host twin, bit for bit; frame-B rows come out unchanged and NaN box
  elements as 0x7fc00000;
- labels: synth.assign_labels with the tolerances of tests/test_assign_gpu.py (ind / mask / cat / gt_boxes exact, hm
  1e-6, anno_box 2e-6), the classes -1 (padding) and len(class_names) ignored.
Edge launches of ops.gt_sample (tests/test_production_datapath_cpu.py builds them): select shared memory just past
48 KB and at the 200 KB cap, one box past the cap (an argument error, every output and workspace byte left as it was), a class call of 70
packed across the collision-row words, zero-point candidates, a scene class len(class_names), a frame without scene
boxes; and one ops.global_aug at 3 x 540k points with all four record kinds and both flips.  Self-checks show that each
comparison fails on a planted error."""
import json
import os
import pickle
import sys
import time
import types

import numpy as np
import pytest
import torch

from oracle import aug_oracle, sweeps_oracle
from oracle import reader_fixtures as RF
from pillarnext_b200 import _lib, hydra_lite, ops, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from test_production_datapath_cpu import (KEYS, SMEM_CAP, SMEM_OPT_IN, aug_launch, boxes_around, grid_launch,  # noqa: E402
                                          gts_fails, gts_oracle_full, same_bits, select_smem, word_launch)
from test_readers_cpu import GOLD, NUSC_TASKS, WAYMO_TASKS, batches, scene_cfg  # noqa: E402

CONFIGS = ("nusc", "waymo")
PT_THREADS, SCAN_CHUNK = 512, 1024        # gt_sample.cu: points per mark / write block, blocks per scan chunk
EXPERIMENT = {"nusc": "nusc_det_pp18_aspp_iou_sp", "waymo": "waymo_det_pp18_aspp_iou_car_sp"}
STAGES = ("accumulate_sweeps", "gt_sample", "global_aug", "assign_labels")

# Entry points the chained stages call, and the test here that checks each one.
COVERED = {
    "pnx_accumulate_sweeps": "test_sweeps_stage_bit_exact",
    "pnx_gt_sample": "test_sampling_stage_bit_exact, test_gt_sample_edge_launches",
    "pnx_global_aug": "test_augmentation_stage_bit_exact, test_global_aug_at_3x540k",
    "pnx_assign_labels": "test_label_stage_matches_numpy",
}
# Host-side workspace queries: they launch nothing (test_every_data_path_entry_point_is_covered checks it).
NO_LAUNCH = ("pnx_accumulate_sweeps_workspace", "pnx_gt_sample_workspace")


# ------------------------------------------------------------------------------------------------- recording
def _relabel(names, frame, rare, common, n_rare, n_outside):
    """A street-like class mix for one frame: n_rare[c] boxes of each rare class c, n_outside names outside the class
    list, the rest cycling through `common`."""
    out, k = [], 0
    for c in rare:
        out += [c] * n_rare[c](frame)
    out += ["animal"] * n_outside
    while len(out) < len(names):
        out.append(common[k % len(common)])
        k += 1
    return np.array(out[:len(names)])


NUSC_RARE = {"truck": lambda f: 1, "construction_vehicle": lambda f: f % 2, "bus": lambda f: 1,
             "trailer": lambda f: 1, "motorcycle": lambda f: 1, "bicycle": lambda f: 1}
WAYMO_RARE = {"pedestrian": lambda f: (12, 2, 8)[f], "cyclist": lambda f: (5, 2, 2)[f]}


def write_tree(name, root):
    """The info tree of config `name` under root, relabelled, and its gt database cut on the GPU."""
    import create_gt_database as tool
    if name == "nusc":
        info = "infos_train_10sweeps_withvelo_filterZero.pkl"
        infos, _ = RF.write_nusc(root, list(range(6)), scene_cfg(NUSC_TASKS, 50.4), n_points=28000, n_boxes=60,
                                 nsweeps=10, nan_velocity=0.2, none_transform=True)
        for f, i in enumerate(infos):
            i["gt_names"] = _relabel(i["gt_names"], f, list(NUSC_RARE), ["car", "car", "pedestrian", "barrier",
                                                                          "traffic_cone", "car", "pedestrian"],
                                     NUSC_RARE, 2)
        db_sweeps = 10
    else:
        info = "waymo_infos_train.pkl"
        infos = RF.write_waymo(root, list(range(3)), scene_cfg(WAYMO_TASKS, 40.0), n_points=200000, n_boxes=150,
                                 nsweeps=3)
        for f, i in enumerate(infos):
            names = _relabel([o["label"] for o in i["objects"]], f, list(WAYMO_RARE), ["vehicle"], WAYMO_RARE, 0)
            for o, n in zip(i["objects"], names):
                o["label"] = str(n)
        db_sweeps = 1
    with open(os.path.join(root, info), "wb") as fh:
        pickle.dump(infos, fh)
    tool.create_reader_database("NUSC" if name == "nusc" else "WAYMO", root, info, nsweeps=db_sweeps,
                                host=not torch.cuda.is_available())
    return info


def experiment(name, root, config_dir):
    """The reference's composed experiment for config `name`, with root_path at the tree."""
    import yaml
    os.makedirs(config_dir, exist_ok=True)
    with open(os.path.join(config_dir, EXPERIMENT[name] + ".yaml"), "w") as fh:
        yaml.safe_dump(json.loads(str(np.load(GOLD)["cfg_" + EXPERIMENT[name]])), fh)
    return hydra_lite.main(config_dir, EXPERIMENT[name], ["data.train_dataset.root_path=" + root])


def draw_batch(name, cfg, seed=11):
    """One collated batch of every frame of the tree through the experiment's training dataset."""
    node = dict(cfg.data.train_dataset)
    if name == "nusc":
        node["resampling"] = False                 # frames in info order, each once
    else:
        node["drop_frames"] = 0.0                  # every past sweep present: 540k points per frame
    np.random.seed(seed)                           # the sampler shuffles its class lists when it is built
    ds = hydra_lite.instantiate(node)
    return batches(ds, len(ds), len(ds), seed)[0]


class _Stop(Exception):
    """Raised by the _forward stub: the chained stages are the code under test."""


class Recorder:
    def __init__(self, real):
        self.real, self.called, self.calls = real, [], {s: [] for s in STAGES}

    def proxy(self):
        rec = self

        class Proxy:
            def __getattr__(self, name):
                if name.startswith("pnx_"):
                    rec.called.append(name)
                return getattr(rec.real, name)
        return Proxy()


def _host(x):
    return x.detach().cpu().numpy().copy() if torch.is_tensor(x) else x


def _wrappers(rec):
    real = {n: getattr(ops, n) for n in STAGES}

    def wrap(n):
        def f(*a, **kw):
            a_host = [_host(x) for x in a]
            out = real[n](*a, **kw)
            rec.calls[n].append((a_host, kw, out))
            return out
        return f
    return {n: wrap(n) for n in STAGES}


def record(name, root):
    """(recorded stage calls, batch, cfg, pnx_* called) of one chained training_step of config `name`."""
    from pillarnext_b200.trainer import example_to_device
    info = write_tree(name, root)
    cfg = experiment(name, root, os.path.join(root, "configs"))
    batch = draw_batch(name, cfg)
    assert info and "sweep_points" in batch and "gts_boxes" in batch and "aug" in batch
    torch.manual_seed(0)
    model = hydra_lite.instantiate(cfg.model).cuda().train()
    rec = Recorder(_lib.lib())
    with pytest.MonkeyPatch.context() as mp:
        proxy = rec.proxy()
        mp.setattr(_lib, "lib", lambda: proxy)
        mp.setattr(ops, "lib", lambda: proxy)
        for n, f in _wrappers(rec).items():
            mp.setattr(ops, n, f)

        def stop(*a, **kw):
            raise _Stop()
        mp.setattr(model, "_forward", stop)
        with pytest.raises(_Stop):
            model.training_step(example_to_device(batch, torch.device("cuda")))
    torch.cuda.synchronize()
    out = {n: [(a, kw, tuple(_host(o) for o in (r if isinstance(r, tuple) else (r,)))) for a, kw, r in rec.calls[n]]
           for n in STAGES}
    # assign_labels returns a dict of per-task lists
    out["assign_labels"] = [(a, kw, {k: [_host(t) for t in v] for k, v in r[0].items()})
                            for a, kw, r in out["assign_labels"]]
    del model
    return types.SimpleNamespace(name=name, calls=out, batch=batch, called=set(rec.called))


T0 = {}


@pytest.fixture(scope="module")
def steps(tmp_path_factory):
    T0["t"] = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    out = {}
    for name in CONFIGS:
        t = time.perf_counter()
        out[name] = record(name, str(tmp_path_factory.mktemp(name)))
        print("\n%s: recorded in %.1f s, peak %.2f GB" % (name, time.perf_counter() - t,
                                                         torch.cuda.max_memory_allocated() / 2 ** 30))
    return out


def _one(r, stage):
    assert len(r.calls[stage]) == 1, (r.name, stage, len(r.calls[stage]))
    return r.calls[stage][0]


# ------------------------------------------------------------------------------------------------- shapes
def _longest_call(classes):
    """Length of the longest class call (run of one class id >= 0) in one frame's candidate classes."""
    best = run = 0
    for k, c in enumerate(classes):
        run = run + 1 if c >= 0 and k > 0 and c == classes[k - 1] else int(c >= 0)
        best = max(best, run)
    return best


def test_recorded_batches_reach_the_production_shapes(steps):
    for name in CONFIGS:
        r = steps[name]
        (a, _, (pts_out, boxes_out, cls_out, accepted, count)) = _one(r, "gt_sample")
        n, B = len(a[0]), a[1].shape[0]
        nblk = -(-n // PT_THREADS)
        tail = int((a[0][:, 0] == B).sum())
        acc = accepted.astype(bool)
        real = a[5] >= 0
        n_acc, n_rej = (acc & real).sum(1), (~acc & real).sum(1)
        M, S = a[1].shape[1], a[4].shape[1]
        longest = max(_longest_call(c) for c in a[5])
        print("%-5s gt_sample: %d points in %d blocks = %d scan chunks, %d frame-B tail rows in; M + S = %d (%d bytes of "
              "select shared memory), longest class call %d; accepted per frame %s, rejected %s; NaN box elements %d" % (
                  name, n, nblk, -(-nblk // SCAN_CHUNK), tail, M + S, select_smem(M, S), longest, n_acc.tolist(),
                  n_rej.tolist(), int(np.isnan(a[1]).sum())))
        assert nblk > 3 * SCAN_CHUNK, (name, nblk)
        assert (n_acc > 0).all() and (n_rej > 0).all(), (name, n_acc, n_rej)
        if name == "nusc":             # min_distance 1 m drops close sweep points: their rows come as frame B
            assert tail > 0 and np.isnan(a[1][..., 6:8]).any()
            cls = _one(r, "assign_labels")[0][1]
            assert (cls == -1).any() and (cls == sum(len(t) for t in NUSC_TASKS)).any()


# ------------------------------------------------------------------------------------------------- stages
def test_sweeps_stage_bit_exact(steps):
    bad = []
    for name in CONFIGS:
        a, _, (out, count) = _one(steps[name], "accumulate_sweeps")
        want, wcount = sweeps_oracle.accumulate(*a)
        host, hcount = ops.accumulate_sweeps_host(*a)
        for what, w, c in (("oracle", want, wcount), ("host twin", host, hcount)):
            if not same_bits(out, w) or int(count[0]) != c:
                diff = np.flatnonzero((out != w).any(1)) if out.shape == w.shape else []
                bad.append("%s sweeps vs %s: count %d / %d, %d rows differ, first %s" % (
                    name, what, int(count[0]), c, len(diff), diff[:5]))
        print("%-5s sweeps: %d key + %d sweep points -> %d rows, count %d" % (name, len(a[0]), len(a[2]), len(out), c))
    assert not bad, bad


def _gts_refs(a):
    return gts_oracle_full(dict(zip(KEYS, a))), ops.gt_sample_host(*a)


def test_sampling_stage_bit_exact(steps):
    bad = []
    for name in CONFIGS:
        a, _, got = _one(steps[name], "gt_sample")
        want, host = _gts_refs(a)
        bad += gts_fails(got, want, name + " gt_sample vs oracle") + gts_fails(got, host, name + " gt_sample vs host twin")
        B, c = a[1].shape[0], int(got[4][0])
        tail = got[0][c:]
        if not ((tail[:, 0] == B).all() and (tail[:, 1:] == 0).all()):
            bad.append("%s: rows past count are not (B, 0, ...)" % name)
        steps[name].gts_want = want
    assert not bad, bad


def test_augmentation_stage_bit_exact(steps):
    bad = []
    for name in CONFIGS:
        (p, b, aug), _, (po, bo) = _one(steps[name], "global_aug")
        B = b.shape[0]
        want = aug_oracle.apply(p, b, aug)
        host = ops.global_aug_host(p, b, aug)
        for what, (wp, wb) in (("oracle", want), ("host twin", host)):
            if not (same_bits(po, wp) and same_bits(bo, wb)):
                bad.append("%s global_aug vs %s differs" % (name, what))
        tail = p[:, 0] == B
        if not same_bits(po[tail], p[tail]):
            bad.append("%s: frame-B rows changed" % name)
        nan = np.isnan(b)
        if not (np.isnan(bo) == nan).all() or not (bo.view(np.int32)[nan] == 0x7fc00000).all():
            bad.append("%s: NaN box elements not kept as 0x7fc00000" % name)
        print("%-5s global_aug: %d points (%d frame B), %d NaN box elements" % (name, len(p), int(tail.sum()), int(nan.sum())))
    assert not bad, bad


def _label_cfg(a):
    _, _, tasks, vs, pr, osf = a
    return dict(tasks=[list(t) for t in tasks], voxel_size=list(vs), pc_range=list(pr), out_size_factor=list(osf))


def assign_fails(got, boxes, cls, cfg, kw, what):
    """pnx_assign_labels against synth.assign_labels: ind / mask / cat exact, hm 1e-6, anno_box 2e-6, gt_boxes exact;
    classes outside [0, len(class_names)) are ignored."""
    names_all = [n for t in cfg["tasks"] for n in t]
    want = [synth.assign_labels(boxes[b], [names_all[c] if 0 <= c < len(names_all) else "ignored_class" for c in cls[b]],
                                cfg=cfg, **kw) for b in range(len(boxes))]
    bad = []
    for t in range(len(cfg["tasks"])):
        for key, tol in (("ind", None), ("mask", None), ("cat", None), ("hm", 1e-6), ("anno_box", 2e-6), ("gt_boxes", 0.0)):
            w, g = np.stack([want[b][key][t] for b in range(len(want))]), got[key][t]
            if g.shape != w.shape or g.dtype != w.dtype:
                bad.append("%s task %d: %s shape / dtype" % (what, t, key))
            elif tol is None:
                if not np.array_equal(g, w):
                    bad.append("%s task %d: %s differs" % (what, t, key))
            else:
                d = np.where(np.isnan(g) & np.isnan(w), 0, np.abs(g.astype(np.float64) - w))
                if np.isnan(d).any() or d.max(initial=0) > tol:
                    bad.append("%s task %d: %s off by %.3g (tolerance %g)" % (what, t, key, np.nanmax(d), tol))
    return bad


def test_label_stage_matches_numpy(steps):
    bad = []
    for name in CONFIGS:
        a, kw, got = _one(steps[name], "assign_labels")
        bad += assign_fails(got, a[0], a[1], _label_cfg(a), kw, name)
        print("%-5s assign_labels: %d frames x %d boxes, positives per task %s" % (
            name, a[0].shape[0], a[0].shape[1], [int(m.sum()) for m in got["mask"]]))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------- edge launches
def _launch_gts(op):
    dev = [torch.from_numpy(op[k]).cuda() for k in KEYS]
    out = ops.gt_sample(*dev)
    torch.cuda.synchronize()
    return tuple(o.cpu().numpy() for o in out)


SENTINEL = 0x5A                            # byte every output and workspace buffer is filled with


def _gt_sample_into_sentinels(op):
    """pnx_gt_sample called directly with every output and the workspace filled with SENTINEL bytes -> (return code,
    error string, whether every byte of them still holds SENTINEL after the device has synchronised).  Each of the four
    kernels writes one of these buffers, so untouched buffers mean nothing was launched."""
    p, b, c, t, cb, cc, ct, cp, co = [torch.from_numpy(op[k]).cuda() for k in KEYS]
    n, (B, M), S, P = len(p), b.shape[:2], cb.shape[1], len(cp)
    L = _lib.lib()
    nbytes = [(n + P) * 6 * 4, B * (M + S) * 9 * 4, B * (M + S) * 4, B * S * 4, 4, max(4, L.pnx_gt_sample_workspace(n, B, S))]
    bufs = [torch.full((k,), SENTINEL, dtype=torch.uint8, device="cuda") for k in nbytes]
    torch.cuda.synchronize()
    rc = L.pnx_gt_sample(p.data_ptr(), n, *[x.data_ptr() for x in (b, c, t)], B, M, *[x.data_ptr() for x in (cb, cc, ct)],
                         S, cp.data_ptr(), co.data_ptr(), P, *[x.data_ptr() for x in bufs], _lib.stream())
    err = L.pnx_last_error().decode() if rc else ""
    torch.cuda.synchronize()
    return rc, err, all(bool((x == SENTINEL).all()) for x in bufs)


def test_gt_sample_edge_launches():
    S = 64
    past48, cap = boxes_around(SMEM_OPT_IN, S)[1], boxes_around(SMEM_CAP, S)[0]
    cases = {"M + S just past 48 KB": grid_launch(past48, S), "M + S at the 200 KB cap": grid_launch(cap, S)}
    word, word_acc = word_launch()
    cases["70-candidate call across the words"] = word
    bad = []
    for what, op in cases.items():
        got = _launch_gts(op)
        want = gts_oracle_full(op)
        host = ops.gt_sample_host(*[op[k] for k in KEYS])
        bad += gts_fails(got, want, what + " vs oracle") + gts_fails(got, host, what + " vs host twin")
        M, Sx = op["gt_boxes"].shape[1], op["cand_boxes"].shape[1]
        print("%s: M + S = %d, select shared memory %d bytes; accepted %d of %d candidates, count %d" % (
            what, M + Sx, select_smem(M, Sx), int(got[3].sum()), int((op["cand_classes"] >= 0).sum()), int(got[4][0])))
    if not same_bits(_launch_gts(word)[3], word_acc.astype(np.int32)):
        bad.append("the word-boundary call's acceptance is not the designed one")
    # one box past the cap: the library's argument error, before any launch
    over = grid_launch(cap + 1, S, n_points=1000)
    assert select_smem(cap + 1, S) > SMEM_CAP
    rc, err, untouched = _gt_sample_into_sentinels(over)
    print("M + S = %d (%d bytes): return code %d, %s; outputs and workspace untouched: %s" % (
        cap + 1 + S, select_smem(cap + 1, S), rc, err, untouched))
    assert rc == -1 and "too many boxes per frame" in err, (rc, err)
    assert untouched, "a kernel ran although the call was refused"
    rc, err, untouched = _gt_sample_into_sentinels(grid_launch(cap, S, n_points=1000))
    assert rc == 0 and not untouched, "the sentinel check would not see a launch"
    assert not bad, bad


def test_global_aug_at_3x540k():
    pts, boxes, aug = aug_launch()
    po, bo = ops.global_aug(*[torch.from_numpy(x).cuda() for x in (pts, boxes, aug)])
    po, bo = po.cpu().numpy(), bo.cpu().numpy()
    wp, wb = aug_oracle.apply(pts, boxes, aug)
    hp, hb = ops.global_aug_host(pts, boxes, aug)
    assert {int(c) for c in aug[:, :, 0].ravel()} == {1, 2, 3, 4}
    assert same_bits(po, wp) and same_bits(bo, wb)
    assert same_bits(po, hp) and same_bits(bo, hb)
    tail = pts[:, 0] == 3
    assert tail.sum() > 0 and same_bits(po[tail], pts[tail])
    assert (bo.view(np.int32)[np.isnan(boxes)] == 0x7fc00000).all()
    print("global_aug: %d points, %d boxes, %d NaN elements: bit-exact with the oracle and the host twin" % (
        len(pts), boxes.shape[0] * boxes.shape[1], int(np.isnan(boxes).sum())))


# ------------------------------------------------------------------------------------------------- self-checks
def test_self_checks_fail_on_planted_errors(steps):
    r = steps["nusc"]
    # sampling: two rows swapped across the boundary of scan chunks 1 and 2, one frame's base off by one, one
    # candidate's acceptance flipped
    a, _, got = _one(r, "gt_sample")
    want = getattr(r, "gts_want", None) or gts_oracle_full(dict(zip(KEYS, a)))
    assert not gts_fails(got, want, "as recorded")
    edge = 2 * SCAN_CHUNK * PT_THREADS
    swapped = got[0].copy()
    swapped[[edge - 1, edge]] = swapped[[edge, edge - 1]]
    assert not same_bits(swapped[edge - 1], got[0][edge - 1])
    assert gts_fails((swapped,) + got[1:], want, "swap")
    f1 = np.flatnonzero(got[0][:, 0] == 1)
    shifted = got[0].copy()
    shifted[f1[0] + 1:f1[-1] + 2] = got[0][f1[0]:f1[-1] + 1]
    assert gts_fails((shifted,) + got[1:], want, "base")
    flipped = got[3].copy()
    flipped[0, 0] ^= 1
    assert gts_fails(got[:3] + (flipped,) + got[4:], want, "accepted")
    # sweeps: one frame's base off by one
    sa, _, (sout, scount) = _one(r, "accumulate_sweeps")
    swant, _ = sweeps_oracle.accumulate(*sa)
    k1 = np.flatnonzero(sout[:, 0] == 1)
    sb = sout.copy()
    sb[k1[0] + 1:k1[-1] + 2] = sout[k1[0]:k1[-1] + 1]
    assert same_bits(sout, swant) and not same_bits(sb, swant)
    # augmentation: a frame-B row augmented as if it were frame B - 1
    (p, b, aug), _, (po, bo) = _one(r, "global_aug")
    B = b.shape[0]
    wp, _ = aug_oracle.apply(p, b, aug)
    i = int(np.flatnonzero(p[:, 0] == B)[0])
    planted = po.copy()
    planted[i, 1:], _ = aug_oracle.apply_frame(p[i:i + 1, 1:], b[B - 1], aug[B - 1])
    assert same_bits(po, wp) and not same_bits(planted, wp)
    # labels: one ind slot shifted by one
    la, kw, lab = _one(r, "assign_labels")
    cfg = _label_cfg(la)
    assert not assign_fails(lab, la[0], la[1], cfg, kw, "as recorded")
    t = int(np.argmax([m.sum() for m in lab["mask"]]))
    bent = {k: list(v) for k, v in lab.items()}
    bent["ind"][t] = bent["ind"][t].copy()
    bent["ind"][t][np.nonzero(lab["mask"][t])[0][0], np.nonzero(lab["mask"][t])[1][0]] += 1
    assert assign_fails(bent, la[0], la[1], cfg, kw, "ind")


# ------------------------------------------------------------------------------------------------- completeness
def test_every_data_path_entry_point_is_covered(steps):
    """Every pnx_* the chained stages called is covered here, replayed by a sibling production test, or a workspace
    query -- and those launch nothing."""
    from test_production_rowwise_gpu import ARG_MAPS, GEMM_REPLAYED
    called = set().union(*(steps[n].called for n in CONFIGS))
    print("\nentry points called: %s" % ", ".join(sorted(called)))
    missing = sorted(n for n in called if n not in COVERED and n not in NO_LAUNCH and n not in ARG_MAPS
                     and n not in GEMM_REPLAYED)
    assert not missing, "entry points the data path calls that no production test covers: %s" % missing
    assert set(COVERED) <= called, sorted(set(COVERED) - called)
    # the workspace queries take sizes only -- no device pointer, no stream -- so they cannot enqueue or write anything;
    # they return the layouts gt_sample.cu and sweeps.cu document
    for q in NO_LAUNCH:
        assert _lib._SIGS[q] and all(a is _lib.I for a in _lib._SIGS[q]), (q, _lib._SIGS[q])
    L = _lib.lib()
    for n, B, S in ((1000, 6, 40), (1608255, 6, 23), (1, 1, 1)):
        nblk = -(-n // PT_THREADS)
        assert L.pnx_gt_sample_workspace(n, B, S) == 4 * (B * S * 11 + B * S + 3 * B + 2 * nblk * B + (n + 3) // 4)
        assert L.pnx_accumulate_sweeps_workspace(n, B) == 4 * (2 * nblk + nblk * 16 + B + 1)
    print("wall time of the file %.1f s, peak GPU memory %.2f GB" % (
        time.perf_counter() - T0["t"], torch.cuda.max_memory_allocated() / 2 ** 30))
