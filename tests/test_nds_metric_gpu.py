"""nuScenes detection score on the GPU: pnx_eval_match_center against its host twin (bit for bit), chunked point counting
against one pass, nuscenes_metrics against the sequential oracle, and the accuracy gate of the nuScenes-configured
detector scored with it."""
import math
import os
import sys

import numpy as np
import pytest
import torch

from oracle import nds_fixtures
from oracle import nds_oracle as O
from pillarnext_b200 import evaluate_nuscenes as EN, ops

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_match_kernel_equals_host_twin_on_crowded_frames():
    gts, det, classes = nds_fixtures.make_frames(21, 200, n_points=None, n_labels=80, extent=15.0, fp_per_frame=300)
    pk = EN.pack(gts, det, classes)
    c_d, m_d = EN.run_device(pk)
    c_h, m_h = EN.run_host(pk)
    assert np.array_equal(c_d, c_h)
    assert m_d.shape == (4, len(pk["det_scores"])) and np.array_equal(m_d, m_h), "%s of %d detections differ" % (
        (m_d != m_h).sum(1), m_d.shape[1])
    n = (m_d >= 0).sum(1)
    assert n[0] > 5000 and (np.diff(n) > 0).all()
    # the fixtures' exact threshold distances and equidistant pairs are there to be decided
    d = pk["det_boxes"].astype(np.float64)
    g = pk["gt_boxes"][pk["det_frames"], np.maximum(m_d[3], 0)].astype(np.float64)
    dist = np.sqrt((d[:, 0] - g[:, 0]) ** 2 + (d[:, 1] - g[:, 1]) ** 2)
    for t, th in enumerate(EN.DIST_THS[:3]):
        assert ((m_d[3] >= 0) & (dist == th)).sum() > 20


def test_chunked_point_count_equals_one_pass():
    gts, det, classes = nds_fixtures.make_frames(22, 24, n_points=30000)
    pk = EN.pack(gts, det, classes)

    def count(p, b, c, t):
        return ops.eval_count_points(*(torch.from_numpy(a).cuda() for a in (p, b, c, t))).cpu().numpy()
    one = EN.count_points(pk, count, point_budget=1 << 30)
    chunked = EN.count_points(pk, count, point_budget=70000)             # two frames per chunk
    assert np.array_equal(one, chunked)
    assert np.array_equal(one, EN.run_host(pk)[0])
    assert one.sum() > 24 * 10000 and ((one == 0) & (pk["gt_classes"] >= 0)).sum() > 0


def assert_close(got, want, tol=1e-9):
    for k, v in want.items():
        if k == "per_class":
            for name, pc in v.items():
                assert_close(got[k][name], pc, tol)
            continue
        g = got[k]
        assert (math.isnan(v) and math.isnan(g)) or abs(g - v) <= tol, (k, g, v)


@pytest.mark.parametrize("kw", [dict(n_points=20000), dict(n_points=None, with_attributes=True)])
def test_nuscenes_metrics_equals_oracle(kw):
    gts, det, classes = nds_fixtures.make_frames(23, 6, fp_per_frame=150, **kw)
    got = EN.nuscenes_metrics(gts, {t: {k: torch.as_tensor(v).cuda() for k, v in d.items()} for t, d in det.items()},
                              classes)
    want = O.nuscenes_metrics(gts, det, classes)
    print({k: v for k, v in got.items() if k != "per_class"})
    assert_close(got, want)
    assert 5 < got["mAP"] < 95 and 5 < got["NDS"] < 95


def test_train_nds_experiment_and_gate(tmp_path):
    import importlib.util
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import train as train_tool
    from test_map_gpu import oracle_detections
    from pillarnext_b200 import functional as Fn, hydra_lite, scenes
    from pillarnext_b200.trainer import example_to_device
    spec = importlib.util.spec_from_file_location("pnx_tools_test", os.path.join(ROOT, "tools", "test.py"))
    test_tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(test_tool)
    work = str(tmp_path)
    torch.manual_seed(0)                                        # the weight initialisation, whatever ran before
    name = "synth_det_pp18_aspp_nds"
    overrides = ["trainer.max_epochs=6", "data.train_dataset.n_frames=640", "data.val_dataset.n_frames=24",
                 "dataloader.train.num_workers=0", "dataloader.val.num_workers=0", "dataloader.train.batch_size=4"]
    tr = train_tool.main(["--config-name", name, "--work-dir", work] + overrides)
    assert tr.epoch == 6
    at_end = tr.last_eval["NDS"]
    res = test_tool.main(["--config-name", name, "--work-dir", work, "+load_from=" + os.path.join(work, "epoch_6.pth")] + overrides)
    assert abs(res["NDS"] - at_end) < 1e-6
    cfg = hydra_lite.main(os.path.join(ROOT, "configs", "experiments"), name, overrides)
    val = hydra_lite.instantiate(cfg.data.val_dataset)
    model = tr.model.eval()
    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items()}
    m_oracle = val.evaluation(oracle_detections(cfg, sd, val))

    def product():
        dets = {}
        with torch.no_grad():
            for i0 in range(0, len(val), 4):
                ex = scenes.collate([val[i] for i in range(i0, min(len(val), i0 + 4))])
                dets.update(model(example_to_device(ex, torch.device("cuda"))))
        return val.evaluation(dets)

    m_bf16 = product()
    with Fn.precision("split"):
        m_split = product()
    msg = "NDS / mAP / mATE / mAVE / mAAE on %d held-out scenes: oracle (fp32 CPU) %s | product fp32-grade %s | product bf16 %s" % (
        len(val), *["%.3f / %.3f / %.3f / %.3f / %.3f" % (m["NDS"], m["mAP"], m["mATE"], m["mAVE"], m["mAAE"])
                    for m in (m_oracle, m_split, m_bf16)])
    print(msg)
    assert m_oracle["mAP"] > 5.0, "the detector did not learn the synthetic task: " + msg
    assert abs(m_split["NDS"] - m_oracle["NDS"]) <= 0.1 and abs(m_split["mAP"] - m_oracle["mAP"]) <= 0.1, msg
    assert abs(m_bf16["NDS"] - m_oracle["NDS"]) <= 1.5, msg
