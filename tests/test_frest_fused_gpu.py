"""-m gpu: the f_rest Adam of the fused step with the live byte (gaussian_backward_kernel<MODE_ADAM_LIVE> updates the staged SH rows,
frest_momentum_kernel the rows that are live but had no staged row) against the step without the byte (frest_stream_kernel over
every row). In deterministic mode the two must agree bit for bit in all 6 parameter tensors and 12 moment tensors.

With the regularisers (MODE_REG) the two paths already differ in a few xyz entries of the small-parameter update, independently of the
f_rest Adam; once xyz differs, the SH view directions of the next step do too. That mode is therefore compared after one step, on the
f_rest parameters and moments, which that step computes from identical inputs."""
import numpy as np
import pytest
import torch

import photo_slam_b200.synthetic as syn

pytestmark = pytest.mark.gpu

P_ODD = 30_011   # not a multiple of 128: the last block is partial
W, H = 320, 240


def _scene(P, seed=7):
    cam0 = syn.make_camera(W, H, 260.0, 260.0)
    sc = syn.make_scene(P, cam0, seed=seed)
    sc["xyz"][::3, 0] += 1000.0      # a third of the rows outside both views: never reached
    rng = np.random.default_rng(seed)
    cam1 = syn.make_camera(W, H, 260.0, 260.0, *syn.random_pose(rng, max_angle=0.3, max_trans=0.4))
    return sc, [cam0, cam1]


def _state(m):
    return [t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_]


def _trainers(cuda, sc, cams, mode):
    """Two identical models: A steps with the live byte, B without it (adam_live = NULL: the MODE_ADAM path)."""
    from photo_slam_b200 import trainer
    out = []
    for live in (True, False):
        m = trainer.GaussianModel.from_numpy(sc, cuda)
        m.trainingSetup(trainer.GaussianOptimizationParams())
        if not live:
            m.adamLive = lambda: None
        if mode == "f3d":
            m.computeFilter3D(cams)
        tr = trainer.GaussianTrainer(m, deterministic=True, antialiasing=mode == "aa", filter3d=mode == "f3d")
        if mode == "reg":
            tr.L.psb_trainer_set_regularizers(tr.h, 0.01, 0.01)
        out.append((m, tr))
    return out


@pytest.mark.parametrize("mode", ["base", "depth", "aa", "reg", "f3d", "normal"])
def test_live_step_bit_identical_to_step_without_live_bytes(cuda, mode):
    sc, cams = _scene(P_ODD)
    dcams = [syn.device_camera(c, cuda) for c in cams]
    gts = [torch.from_numpy(syn.target_image(H, W, seed=2 + i)).to(cuda) for i in range(2)]
    kw = {}
    if mode == "depth":
        kw = dict(gt_depth=torch.full((H, W), 4.0, device=cuda), lambda_depth=0.5)
    elif mode == "normal":
        gn = torch.zeros((3, H, W), device=cuda)
        gn[2] = -1.0
        kw = dict(gt_normal=gn, lambda_normal=0.1)
    (ma, ta), (mb, tb) = _trainers(cuda, sc, cams, mode)
    for it in range(1 if mode == "reg" else 6):      # alternating views: rows staged in one step are momentum-only in the next
        k = it % 2
        for tr in (ta, tb):
            tr.trainForOneIteration(dcams[k], gts[k], **kw)
            tr.result()
    torch.cuda.synchronize()
    live = ma.adam_live_.bool()
    assert 0 < live.sum().item() < ma.num_points(), "the scene must leave rows without a gradient"
    compared = (2, 8, 14) if mode == "reg" else range(18)   # f_rest p, m, v | everything
    for i, (a, b) in enumerate(zip(_state(ma), _state(mb))):
        if i in compared:
            assert torch.equal(a, b), f"tensor {i} ({mode}): {(a != b).sum().item()} entries differ"


def test_overflowing_step_leaves_parameters_moments_and_live_bytes_untouched(cuda):
    """A few steps at a small resolution leave live rows and an arena sized for them; the full-resolution view of the same dense
    scene then overflows it. That step (before result() repeats it) must change nothing."""
    from photo_slam_b200 import trainer
    Wb, Hb = 640, 480
    cam_big = syn.make_camera(Wb, Hb, 520.0, 520.0)
    sc = syn.make_scene(60_011, cam_big, seed=3, scale_px=20.0)
    cam_small = syn.make_camera(80, 60, 65.0, 65.0)
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    tr = trainer.GaussianTrainer(m)
    c_small, c_big = syn.device_camera(cam_small, cuda), syn.device_camera(cam_big, cuda)
    gt_small = torch.from_numpy(syn.target_image(60, 80, seed=4)).to(cuda)
    for _ in range(3):
        tr.trainForOneIteration(c_small, gt_small)
        tr.result()
    torch.cuda.synchronize()
    assert m.adam_live_.bool().any()
    before, live_before = _state(m), m.adam_live_.clone()
    tr.trainForOneIteration(c_big, torch.from_numpy(syn.target_image(Hb, Wb, seed=5)).to(cuda))
    torch.cuda.synchronize()
    after, live_after = _state(m), m.adam_live_.clone()
    tr.result()   # reports the overflow and repeats the step with a grown arena: now the state moves
    torch.cuda.synchronize()
    assert tr._overflow_info()[1] >= 1, "the full-resolution step must overflow the arena"
    for i, (a, b) in enumerate(zip(after, before)):
        assert torch.equal(a, b), f"tensor {i} changed on an overflowing step"
    assert torch.equal(live_after, live_before)
    assert not torch.equal(m.xyz_, before[0])
