"""-m gpu: the RGB-D depth term on the data-parallel paths — the NVLink step (psb_dp_step_depth) and the slab pipeline
(psb_trainer_backward_begin_depth -> psb_trainer_backward_slab) — against the fused depth step on one GPU, and (when the box has
>= 2 GPUs) ranks with and without a depth target in one step against the 1-rank step on the summed gradients."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import scene_tensors

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LRS = [0.00032, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]
LAMBDA_DEPTH = 0.1
SLABS = dict(mode="nccl", pipeline=True, nslabs=3)


def _inputs(cuda, P):
    """test_p2p_step_world1_equals_fused_step's scene and view, a random colour target and a target depth with ~10 % holes and
    some negative (invalid) values."""
    wh = (320, 240)
    cam, sc, act, g, c = scene_tensors(P, "tum", seed=5, pose_seed=6, dev=cuda, wh=wh, scale_px=4.0)
    gt = torch.rand((3, wh[1], wh[0]), generator=torch.Generator().manual_seed(7)).to(cuda)
    V = cam["viewmatrix"].reshape(-1)
    z = sc["xyz"] @ V[[2, 6, 10]] + V[14]
    zs = np.quantile(z[z > 0.2], [0.1, 0.9])
    gen = torch.Generator().manual_seed(11)
    depth = zs[0] + (zs[1] - zs[0]) * torch.rand((wh[1], wh[0]), generator=gen)
    r = torch.rand((wh[1], wh[0]), generator=gen)
    depth[r < 0.1] = 0.0
    depth[(r >= 0.1) & (r < 0.12)] = -1.0
    return sc, c, gt, depth.float().contiguous().to(cuda)


def _model(sc, cuda):
    from photo_slam_b200 import trainer
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    return m


def _finish(tr):
    if hasattr(tr, "sync"):
        tr.sync()
    torch.cuda.synchronize()


def _assert_same_state(a, b, what=""):
    """test_p2p_step_world1_equals_fused_step's tolerances: parameters within half an Adam step (all but 2e-3 of the entries),
    moments within 1e-4 relative norm, densification statistics equal."""
    from photo_slam_b200 import trainer
    for x, y, lr, name in zip(a.tensors(), b.tensors(), LRS, trainer.GROUPS):
        frac = ((x - y).abs() > 0.5 * lr).float().mean().item()
        assert frac < 2e-3, (what, name, frac)
    for x, y in zip(a.exp_avg_ + a.exp_avg_sq_, b.exp_avg_ + b.exp_avg_sq_):
        rn = ((x.double() - y.double()).norm() / (x.double().norm() + 1e-30)).item()
        assert rn < 1e-4, (what, rn)
    for x, y in zip((a.max_radii2D_, a.denom_), (b.max_radii2D_, b.denom_)):
        assert torch.equal(x, y), what


def _assert_same_result(ra, rb, what=""):
    (la, _, _, da, _), (lb, _, _, db, _) = ra, rb
    assert abs(la - lb) <= 2e-5 * max(1.0, abs(la)), (what, la, lb)
    assert abs(da - db) <= 1e-5 * max(1.0, abs(da)), (what, da, db)


@pytest.mark.parametrize("P", [20_000, 12_345])
def test_p2p_depth_step_world1_equals_fused_depth_step(cuda, P):
    from photo_slam_b200 import trainer
    sc, c, gt, gd = _inputs(cuda, P)
    a, b = _model(sc, cuda), _model(sc, cuda)
    ta, tb = trainer.GaussianTrainer(a), trainer.DataParallelTrainer(b, mode="p2p")
    assert tb.mode == "p2p"
    for it in range(4):
        ta.trainForOneIteration(c, gt, gt_depth=gd, lambda_depth=LAMBDA_DEPTH)
        tb.trainForOneIteration(c, gt, gt_depth=gd, lambda_depth=LAMBDA_DEPTH)
        ra, rb = ta.result_depth(), tb.result_depth()
        assert ra[3] > 0.0
        _assert_same_result(ra, rb, it)
    _finish(tb)
    assert tb.status() == 0
    _assert_same_state(a, b)
    tb.close()


def test_slab_pipeline_depth_step_equals_flat_split_and_fused_depth_steps(cuda):
    from photo_slam_b200 import trainer
    sc, c, gt, gd = _inputs(cuda, 12_345)
    models = [_model(sc, cuda) for _ in range(3)]
    trs = [trainer.DataParallelTrainer(models[0], **SLABS), trainer.DataParallelTrainer(models[1], mode="nccl", pipeline=False),
           trainer.GaussianTrainer(models[2])]
    assert trs[0].pipeline and not trs[1].pipeline
    for it in range(3):
        res = []
        for tr in trs:
            tr.trainForOneIteration(c, gt, gt_depth=gd, lambda_depth=LAMBDA_DEPTH)
            res.append(tr.result_depth())
        _assert_same_result(res[0], res[1], ("flat", it))
        _assert_same_result(res[0], res[2], ("fused", it))
    torch.cuda.synchronize()
    # the split paths keep no adam_live bytes, and both of them reduce their gradients in the same order
    _assert_same_state(models[0], models[1], "flat")
    _assert_same_state(models[2], models[0], "fused")


def _render_target(tr, c):
    """the current render of the trainer's own model: with lambda_dssim = 0 its photometric gradient is exactly zero"""
    img = tr.render(c)
    torch.cuda.synchronize()
    return img.clone()


@pytest.mark.parametrize("kw", [dict(mode="p2p"), SLABS], ids=["p2p", "slabs"])
def test_plain_steps_between_depth_steps_leave_no_stale_depth_gradient(cuda, kw):
    """depth, plain, depth, plain, depth with every colour target equal to the render: each depth step reaches its rows through
    dL/dz alone. If any per-Gaussian kernel that follows a depth tile backward ignored slot 11, dL/dz would be lost from its own
    step and added to the next depth step; the sequence must equal the same sequence of fused steps."""
    from photo_slam_b200 import trainer
    sc, c, gt, gd = _inputs(cuda, 12_345)
    a, b = _model(sc, cuda), _model(sc, cuda)
    ta, tb = trainer.GaussianTrainer(a), trainer.DataParallelTrainer(b, **kw)
    for tr in (ta, tb):
        tr.opt.lambda_dssim = 0.0
    for it, with_depth in enumerate((True, False, True, False, True)):
        dkw = dict(gt_depth=gd, lambda_depth=LAMBDA_DEPTH) if with_depth else dict()
        res = []
        for tr in (ta, tb):
            tr.trainForOneIteration(c, _render_target(tr, c), **dkw)
            res.append(tr.result_depth())
        assert res[0][1] == 0.0 and res[1][1] == 0.0, "the colour target must equal the render"
        assert (res[0][3] > 0.0) == with_depth
        _assert_same_result(res[0], res[1], it)
    _finish(tb)
    _assert_same_state(a, b)
    tb.close()


def test_p2p_depth_only_rows_are_updated_like_the_fused_step(cuda):
    """Every colour target equals the render and lambda_dssim = 0: only dL/dz reaches the rows, and the records carry it."""
    from photo_slam_b200 import trainer
    sc, c, gt, gd = _inputs(cuda, 20_000)
    a, b = _model(sc, cuda), _model(sc, cuda)
    ta, tb = trainer.GaussianTrainer(a), trainer.DataParallelTrainer(b, mode="p2p")
    before = a.xyz_.clone()
    for tr in (ta, tb):
        tr.opt.lambda_dssim = 0.0
        tr.trainForOneIteration(c, _render_target(tr, c), gt_depth=gd, lambda_depth=LAMBDA_DEPTH)
    ra, rb = ta.result_depth(), tb.result_depth()
    _finish(tb)
    assert ra[1] == 0.0 and rb[1] == 0.0 and rb[3] > 0.0
    _assert_same_result(ra, rb)
    moved_a, moved_b = (a.xyz_ != before).any(dim=1), (b.xyz_ != before).any(dim=1)
    assert moved_b.sum().item() > 100
    assert (moved_a != moved_b).sum().item() <= 2e-3 * moved_a.numel()
    rows = moved_a & moved_b
    frac = ((a.xyz_[rows] - b.xyz_[rows]).abs() > 0.5 * LRS[0]).float().mean().item()
    assert frac < 2e-3, frac
    _assert_same_state(a, b)
    tb.close()


@pytest.mark.parametrize("kw", [dict(mode="p2p"), SLABS], ids=["p2p", "slabs"])
def test_overflowing_depth_view_is_dropped_not_retried(cuda, kw):
    """test_overflowing_view_is_dropped_not_retried_on_the_data_parallel_path with a depth target: the view contributes a zero
    gradient, result_depth() is all NaN, and the next depth step of the same view trains."""
    from photo_slam_b200 import trainer
    P, wh = 2_000, (640, 480)
    cam, sc, act, g, c = scene_tensors(P, "tum", seed=2, pose_seed=None, dev=cuda, wh=wh, scale_px=150.0)
    gt = torch.rand((3, wh[1], wh[0]), device=cuda)
    gd = torch.rand((wh[1], wh[0]), device=cuda) * 4.0
    m = _model(sc, cuda)
    tr = trainer.DataParallelTrainer(m, **kw)
    before = [t.clone() for t in m.tensors()]
    tr.trainForOneIteration(c, gt, gt_depth=gd, lambda_depth=LAMBDA_DEPTH)
    res = tr.result_depth()
    _finish(tr)
    assert res[4] > 6 * P + 65536 and tr.dropped_views == 1
    assert all(x != x for x in res[:4]), res
    for x, y in zip(before, m.tensors()):
        assert torch.equal(x, y), "a dropped view must not move the parameters (zero gradient, zero moments)"
    assert not any(t.any() for t in m.exp_avg_ + m.exp_avg_sq_)
    tr.trainForOneIteration(c, gt, gt_depth=gd, lambda_depth=LAMBDA_DEPTH)
    res2 = tr.result_depth()
    _finish(tr)
    assert res2[0] == res2[0] and res2[3] > 0.0 and tr.dropped_views == 1
    assert not torch.equal(before[0], m.xyz_)
    tr.close()


def test_p2p_train_host_with_depth_equals_device_inputs(cuda):
    from photo_slam_b200 import trainer
    sc, c, gt, gd = _inputs(cuda, 12_345)
    a, b = _model(sc, cuda), _model(sc, cuda)
    ta, tb = trainer.DataParallelTrainer(a, mode="p2p"), trainer.DataParallelTrainer(b, mode="p2p")
    pin = lambda t: t.cpu().pin_memory()
    host_cam = dict(c, viewmatrix=pin(c["viewmatrix"]), projmatrix=pin(c["projmatrix"]), campos=pin(c["campos"]))
    host_gt, host_depth = pin(gt), pin(gd)
    for it in range(3):
        ta.trainForOneIteration(c, gt, gt_depth=gd, lambda_depth=LAMBDA_DEPTH)
        la = ta.result()[0]
        lb = tb.trainHost(host_cam, host_gt, host_depth=host_depth, lambda_depth=LAMBDA_DEPTH)
        assert abs(la - lb) <= 2e-5 * max(1.0, abs(la)), (it, la, lb)
    tb.flushHost()
    _finish(ta)
    _finish(tb)
    _assert_same_state(a, b)
    ta.close()
    tb.close()


def _launch(world, mode, P, steps=3, timeout=420):
    port = 29500 + ((os.getpid() + 200) % 400)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "dp_depth_worker.py"), mode, str(P), str(steps)]
    env = dict(os.environ, PSB_DP_TIMEOUT_MS="15000")
    return subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_multi_rank_mixed_depth_replicas_identical_and_equal_summed_gradient_step(cuda, mode):
    """Even ranks train with a depth target, odd ranks without (mode="nccl" runs the slab pipeline at world > 1)."""
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 4 else (4 if n < 8 else 8)
    r = _launch(world, mode, 30_001)
    assert r.returncode == 0 and "DP_DEPTH_WORKER_OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
    print(r.stdout.strip().splitlines()[-1])
