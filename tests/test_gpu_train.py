"""GPU parity of the training path: train-mode LiDARModel forward/backward (CUDA pillar decorate + scatter-max with
arg-routed backward, batch-stat BatchNorm) against the REFERENCE loss/gradients stored in tests/golden."""
import os

import numpy as np
import pytest
import torch

from lav_b200 import synth
from tests import util

pytestmark = pytest.mark.gpu


def test_train_forward_backward_matches_reference_golden(cuda, golden_dir):
    gold = np.load(os.path.join(golden_dir, "lidar_model_train.npz"))
    m, _ = util.lidar_model(cuda)
    m.train()
    clouds = [c.to(cuda) for c in util.pillar_clouds()]
    outs = m(clouds, [len(c) for c in clouds])
    names = ["features", "center", "box", "ori", "seg"]
    for n, o in zip(names, outs):
        assert util.rel_err(o.detach()[:, :, ::8, ::8], torch.from_numpy(gold["out_" + n])) < 1e-3, n
    gw = [torch.randn(o.shape, generator=synth._gen(7, f"gw{i}")).to(cuda) for i, o in enumerate(outs)]
    loss = sum((o * g).sum() for o, g in zip(outs, gw)) / 1e3
    assert abs(float(loss) - float(gold["loss"])) < 1e-3 * abs(float(gold["loss"])) + 1e-3
    loss.backward()
    # Every parameter gradient against the REFERENCE's digest (l2 norm, projection on a seeded vector).  Deep-layer
    # gradients of this untrained, batch-stat-BN network are ill-conditioned: the oracle itself, run on another CPU,
    # moves by 1e-3..1e-2 of the gradient norm (scripts/train_debug.py), so the gate is
    # statistical for the trunk and tight for the output layers, whose gradients do not pass through the trunk.
    import json
    dig = json.load(open(os.path.join(golden_dir, "lidar_model_train_grad_digest.json")))
    for k, p in m.named_parameters():
        g = p.grad.detach().cpu()
        n0, s0, p0, mx = dig[k]
        if n0 < 1e-3:        # e.g. the Linear bias in front of a batch-stat BatchNorm: its true gradient is 0, the rest is noise
            continue
        r = torch.randn(g.shape, generator=synth._gen(13, "dg:" + k))
        shallow = "_head.net.2." in k or "_head.net.3." in k
        assert abs(float(g.norm()) / n0 - 1) < (1e-4 if shallow else 1e-2), (k, float(g.norm()), n0)
        assert abs(float((g * r).sum()) - p0) / n0 < (2e-4 if shallow else 3e-2), (k, float((g * r).sum()), p0, n0)
    grads = dict(m.named_parameters())
    for key in gold.files:
        if key.startswith("grad:"):
            assert util.rel_err(grads[key[5:]].grad, torch.from_numpy(gold[key])) < 8e-2, key


def test_perception_trainer_step_decreases_loss(cuda):
    from lav_b200.train import PerceptionTrainer
    m, _ = util.lidar_model(cuda)
    tr = PerceptionTrainer(m, lr=1e-3, device=cuda)
    clouds = [c.to(cuda) for c in util.pillar_clouds()]
    g = synth._gen(3, "tgt")
    heat = (torch.rand(2, 2, 320, 320, generator=g) > 0.995).float().to(cuda)
    size = torch.rand(2, 2, 320, 320, generator=g).to(cuda)
    ori = torch.randn(2, 2, 320, 320, generator=g).to(cuda)
    bev = (torch.rand(2, 9, 320, 320, generator=g) > 0.5).float().to(cuda)
    losses = [float(tr.train_step(clouds, [len(c) for c in clouds], heat, size, ori, bev)[0]) for _ in range(6)]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0]


def test_full_train_lidar_step(cuda):
    """LAVTrainer.train_lidar: LiDAR model + UniPlanner student vs frozen teacher, all 8 losses finite, parameters move,
    the teacher stays frozen."""
    from lav_b200.train import LAVTrainer, synthetic_train_batch
    from tests.test_heads_cpu import uniplanner
    m, _ = util.lidar_model(cuda)
    up, _ = uniplanner()
    up = up.to(cuda)
    tr = LAVTrainer(m, up, lr=1e-4, device=cuda)
    batch = synthetic_train_batch(2, cuda, n_points=(20000, 30000))
    teacher0 = [p.detach().clone() for p in up.bev_planner.parameters()]
    w0 = up.plan_mlp.weight.detach().clone()
    l0, parts = tr.train_lidar(*batch)
    l1, _ = tr.train_lidar(*batch)
    assert all(torch.isfinite(v) for v in parts.values()) and torch.isfinite(l0) and torch.isfinite(l1)
    assert set(parts) == {"hm_loss", "box_loss", "ori_loss", "seg_loss", "plan_loss", "ego_cast_loss", "other_cast_loss", "cmd_loss"}
    assert not torch.equal(w0, up.plan_mlp.weight)
    assert all(torch.equal(a, b) for a, b in zip(teacher0, up.bev_planner.parameters()))
