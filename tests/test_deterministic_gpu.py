"""-m gpu: deterministic mode (psb_trainer_set_deterministic; GaussianTrainer / DataParallelTrainer(deterministic=True)).

  * repeat runs: fresh contexts with the mode on, the same seeded model and the same calls end with every parameter, moment,
    statistic, exist_since_iter, image, radii and loss scalar bit-identical (torch.equal), over steps with a mask, an SH-degree
    change, a depth target on some steps and one Philox densification in the middle;
  * an arena that overflows and is grown on the retry path ends where a pre-grown arena ends;
  * psb_trainer_backward gradients are bit-identical run to run and equal to the gradients assembled from
    psb_trainer_backward_begin + every psb_trainer_backward_slab;
  * against the stored reference outputs the mode passes the per-element gates of test_trainer_parity_gpu.py, and its gradients
    match the default mode's;
  * the NVLink step (psb_dp_step) is bit-identical run to run at world 1 (with and without depth) and, on a multi-GPU box, across
    ranks and runs;
  * the operator path, which has no deterministic backward, raises under torch.use_deterministic_algorithms(True).
"""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

from helpers import SAMPLE, Gold, rel_close, scene_tensors

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WH = (600, 340)
LAMBDA_DEPTH = 0.1


def _inputs(cuda, P, scale_px, seed=3):
    cam, sc, act, g, c = scene_tensors(P, "replica", seed=seed, pose_seed=seed + 1, dev=cuda, wh=WH, scale_px=scale_px)
    W, H = WH
    gen = torch.Generator().manual_seed(seed + 2)
    gt = torch.rand((3, H, W), generator=gen).to(cuda)
    mask = torch.ones((3, H, W))
    mask[:, 40:120, 100:260] = 0.0
    depth = 0.5 + 7.5 * torch.rand((H, W), generator=gen)
    depth[torch.rand((H, W), generator=gen) < 0.1] = 0.0
    return sc, c, gt, mask.to(cuda), depth.to(cuda)


def _model(sc, cuda):
    from photo_slam_b200 import trainer
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    m.setShDegree(1)
    return m


def _state(m):
    return [t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + [m.xyz_gradient_accum_, m.denom_, m.max_radii2D_, m._exist()]]


def _train_run(cuda, inputs, steps=20, densify_at=10):
    """One fused-step run with the mode on: every step's image, radii and result_depth(), and the final model state."""
    from photo_slam_b200 import trainer
    sc, c, gt, mask, gd = inputs
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m, deterministic=True)
    H, W = c["H"], c["W"]
    images, radii, results = [], [], []
    for it in range(steps):
        if it == 6:
            m.oneUpShDegree()
        if it == densify_at:
            counts = m.densifyAndPrune(1e-6, 0.005, 5.0, 0, seed=7, offset=it)
            assert counts[2] + counts[4] > 0, counts        # clones and splits happened
        img = torch.empty((3, H, W), device=cuda)
        rad = torch.empty(m.num_points(), dtype=torch.int32, device=cuda)
        dkw = dict(gt_depth=gd, lambda_depth=LAMBDA_DEPTH) if it % 3 == 1 else {}
        tr.trainForOneIteration(c, gt, mask if it % 2 == 0 else None, out_color=img, radii=rad, **dkw)
        results.append(tr.result_depth())
        images.append(img)
        radii.append(rad)
    torch.cuda.synchronize()
    return dict(images=images, radii=radii, results=results, state=_state(m))


def _same_scalars(a, b):
    """bit-for-bit (repr of a float is exact; a dropped data-parallel view reports NaN)"""
    return repr(a) == repr(b)


def _assert_equal_runs(a, b):
    assert _same_scalars(a["results"], b["results"]), "loss scalars differ"
    assert all(torch.equal(x, y) for x, y in zip(a["images"], b["images"])), "rendered images differ"
    assert all(torch.equal(x, y) for x, y in zip(a["radii"], b["radii"])), "radii differ"
    assert len(a["state"]) == len(b["state"])
    for i, (x, y) in enumerate(zip(a["state"], b["state"])):
        assert x.shape == y.shape and torch.equal(x, y), f"model state tensor {i} differs"


def test_repeat_runs_are_bit_identical(cuda):
    inputs = _inputs(cuda, 200_000, 6.0)
    a = _train_run(cuda, inputs)
    r0 = a["radii"][0]
    assert int((r0 >= 16).sum()) > 10_000, "want many Gaussians over 3 or more tiles"
    assert a["state"][0].size(0) > 200_000 and any(r[3] > 0 for r in a["results"])
    b = _train_run(cuda, inputs)
    _assert_equal_runs(a, b)
    c = _train_run(cuda, inputs)
    _assert_equal_runs(a, c)


def test_overflow_retry_ends_bit_identical_to_a_large_enough_arena(cuda):
    """Context A's arena is grown by a render of the view before its first step; context B's first step overflows, reports
    PSB_ERR_RETRY (the slot buffer grows with the arena) and is repeated by result()."""
    from photo_slam_b200 import trainer
    sc, c, gt, mask, gd = _inputs(cuda, 100_000, 20.0, seed=5)
    runs = []
    for pregrow in (True, False):
        m = _model(sc, cuda)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        if pregrow:
            tr.render(c)
        first_overflow = None
        for it in range(4):
            tr.trainForOneIteration(c, gt, mask, **(dict(gt_depth=gd, lambda_depth=LAMBDA_DEPTH) if it % 2 else {}))
            res = tr.result_depth()
            if it == 0:
                first_overflow = tr._overflow_info()
        torch.cuda.synchronize()
        assert res[4] > 6 * 100_000 + 65536, "the view must overflow the initial arena"
        runs.append((first_overflow, res, _state(m)))
    (ov_a, res_a, st_a), (ov_b, res_b, st_b) = runs
    assert ov_a[1] == 1 and ov_a[0] == 1, "A: the render (pass 1) overflowed"
    assert ov_b[1] == 1 and ov_b[0] == 1, "B: the first step (pass 1) overflowed and was retried"
    assert _same_scalars(res_a, res_b)
    for x, y in zip(st_a, st_b):
        assert torch.equal(x, y)


def _backward_grads(tr, m, c, gt, gd=None):
    """psb_trainer_backward(_depth) into a fresh gradient buffer (repeated once if the arena had to grow)."""
    from photo_slam_b200 import _lib, trainer
    from photo_slam_b200.parallel import GradBuffer
    P = m.num_points()
    buf = GradBuffer(P, m.device)
    stream = torch.cuda.current_stream().cuda_stream
    depth = trainer._cdepth(gd, LAMBDA_DEPTH if gd is not None else 0.0, None)
    for attempt in range(2):
        cm, cc, cs = m._cmodel(), trainer._ccamera(c), tr._cstep(True)
        ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in buf.segments])
        args = (tr.h, P, 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(), None, C.byref(cs), None, None, ptrs)
        if depth is None:
            _lib.check(tr.L.psb_trainer_backward(*args, stream), "psb_trainer_backward")
        else:
            _lib.check(tr.L.psb_trainer_backward_depth(*args, C.byref(depth), stream), "psb_trainer_backward_depth")
        out, n = (C.c_float * 4)(), C.c_int()
        rc = tr.L.psb_trainer_result_depth(tr.h, out, C.byref(n), stream)
        if rc == 0:
            break
        assert rc == -4 and attempt == 0, rc
        m.max_radii2D_.zero_(); m.xyz_gradient_accum_.zero_(); m.denom_.zero_()
    torch.cuda.synchronize()
    return buf.flat.clone(), list(out)


def _slab_grads(tr, m, c, gt, gd=None, nslabs=3):
    """psb_trainer_backward_begin_depth + one psb_trainer_backward_slab per slab, written into the flat layout of GradBuffer."""
    from photo_slam_b200 import _lib, trainer
    from photo_slam_b200.parallel import GradBuffer, SlabGradBuffer
    L = tr.L
    P = m.num_points()
    buf = GradBuffer(P, m.device)
    stream = torch.cuda.current_stream().cuda_stream
    depth = trainer._cdepth(gd, LAMBDA_DEPTH if gd is not None else 0.0, None)
    cm, cc, cs = m._cmodel(), trainer._ccamera(c), tr._cstep(True)
    _lib.check(L.psb_trainer_backward_begin_depth(tr.h, P, 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(), None, C.byref(cs),
                                                  None, None, C.byref(depth) if depth is not None else None, stream), "psb_trainer_backward_begin_depth")
    # (the slab call writes row g at grads[i] + g * SIZES[i], see SlabGradBuffer.kernel_pointers: the full segments take every slab)
    ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in buf.segments])
    for first, count in SlabGradBuffer(P, m.device, nslabs).slabs:
        _lib.check(L.psb_trainer_backward_slab(tr.h, P, 16, C.byref(cm), C.byref(cc), C.byref(cs), first, count, ptrs, stream), "psb_trainer_backward_slab")
    out, n = (C.c_float * 4)(), C.c_int()
    assert tr.L.psb_trainer_result_depth(tr.h, out, C.byref(n), stream) == 0
    torch.cuda.synchronize()
    return buf.flat.clone(), list(out)


@pytest.mark.parametrize("with_depth", [False, True], ids=["plain", "depth"])
def test_backward_gradients_bit_identical_and_equal_to_slabs(cuda, with_depth):
    from photo_slam_b200 import trainer
    sc, c, gt, mask, gd = _inputs(cuda, 150_000, 6.0, seed=9)
    gd = gd if with_depth else None
    outs = []
    for _ in range(2):
        m = _model(sc, cuda)
        tr = trainer.DataParallelTrainer(m, mode="nccl", pipeline=False, deterministic=True)
        outs.append(_backward_grads(tr, m, c, gt, gd))
    (ga, la), (gb, lb) = outs
    assert ga.abs().sum() > 0
    assert torch.equal(ga, gb) and _same_scalars(la, lb)
    # the same context again (its arena is now large enough), then begin + slabs
    gc, lc = _backward_grads(tr, m, c, gt, gd)
    gs, ls = _slab_grads(tr, m, c, gt, gd)
    assert torch.equal(ga, gc) and torch.equal(ga, gs) and _same_scalars(la, lc) and _same_scalars(la, ls)


def test_mode_passes_the_reference_gates_and_matches_the_default_mode(cuda):
    """test_trainer_parity_gpu.py's per-element gates against the stored reference outputs (config B at 600x340), with the mode on;
    and the mode's gradients against the default mode's within that test's relative-norm bound."""
    import test_trainer_parity_gpu as tp
    from photo_slam_b200 import trainer
    P, camname, wh = 500_000, "replica", (600, 340)
    r = Gold(tp.MODULE, tp._cid(P, camname, wh))
    sc, c, gt = tp._inputs(P, camname, wh, cuda)
    few = lambda bound: max(bound, 2 / SAMPLE)
    res = {}
    for det in (True, False):
        m = trainer.GaussianModel.from_numpy(sc, cuda)
        m.trainingSetup(trainer.GaussianOptimizationParams())
        tr = trainer.DataParallelTrainer(m, mode="nccl", pipeline=False, deterministic=det)
        flat, out = _backward_grads(tr, m, c, gt)
        from photo_slam_b200.parallel import GradBuffer
        gb = GradBuffer(P, cuda)
        gb.flat.copy_(flat)
        img = torch.empty((3, wh[1], wh[0]), device=cuda)
        radii = torch.empty(P, dtype=torch.int32, device=cuda)
        tr.render(c, out=img, radii=radii)
        torch.cuda.synchronize()
        res[det] = dict(grads=[v.clone() for v in gb.views()], loss=out[0], image=img, radii=radii)
    d = res[True]
    assert abs(d["loss"] - r["loss"]) <= 1e-5 * max(1.0, abs(r["loss"]))
    assert r.frac("image", d["image"], atol=1e-6) <= few(5e-4)
    vis = d["radii"] > 0
    for name, a, b in zip(trainer.GROUPS, d["grads"], res[False]["grads"]):
        a, b = a.reshape(P, -1), b.reshape(P, -1)
        key = "grad_" + name
        scale, self_frac = r[key + "#max"] + 1e-30, r[key + "#self"]
        x, y = r.pair(key, a)
        live = (x != 0) | (y != 0)
        frac = rel_close(x[live], y[live], rtol=1e-4, atol=1e-6 * scale)
        nrm = ((x - y).norm() / (y.norm() + 1e-30)).item()
        print(f"deterministic grad {name}: frac>1e-4 {frac:.2e} (reference vs itself {self_frac:.2e}), rel-norm {nrm:.2e}")
        assert nrm < 2e-4, (name, nrm)
        assert frac <= few(max(1e-3, 3 * self_frac)), (name, frac, self_frac)
        assert not a[~vis].any()
        dn = ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()
        assert dn < 2e-4, f"{name}: deterministic vs default rel-norm {dn}"


@pytest.mark.parametrize("with_depth", [False, True], ids=["plain", "depth"])
def test_p2p_world1_bit_identical_run_to_run(cuda, with_depth):
    from photo_slam_b200 import trainer
    sc, c, gt, mask, gd = _inputs(cuda, 60_000, 6.0, seed=13)
    runs = []
    for _ in range(2):
        m = _model(sc, cuda)
        tr = trainer.DataParallelTrainer(m, mode="p2p", deterministic=True)
        assert tr.mode == "p2p"
        tr.render(c)        # grows the binning arena: no step is a dropped view
        results = []
        for it in range(4):
            tr.trainForOneIteration(c, gt, mask, **(dict(gt_depth=gd, lambda_depth=LAMBDA_DEPTH) if with_depth else {}))
            results.append(tr.result_depth())
        tr.sync()
        torch.cuda.synchronize()
        assert tr.status() == 0
        runs.append((results, _state(m)))
        tr.close()
    (ra, sa), (rb, sb) = runs
    assert _same_scalars(ra, rb) and all(r[0] == r[0] for r in ra)
    assert all(torch.equal(x, y) for x, y in zip(sa, sb))


def _launch(world, P, steps=4, timeout=420):
    port = 29500 + ((os.getpid() + 100) % 400)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "dp_deterministic_worker.py"), str(P), str(steps)]
    env = dict(os.environ, PSB_DP_TIMEOUT_MS="15000")
    return subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)


def test_multi_rank_p2p_bit_identical_across_ranks_and_runs(cuda):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 4 else (4 if n < 8 else 8)
    digests = []
    for _ in range(2):
        r = _launch(world, 30_001)
        assert r.returncode == 0 and "DP_DET_WORKER_OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
        line = [x for x in r.stdout.splitlines() if x.startswith("DP_DET_WORKER_OK")][-1]
        print(line)
        digests.append(line.split("digest=")[1].split()[0])
    assert digests[0] == digests[1]


@pytest.fixture
def torch_deterministic_flag():
    before, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(before, warn_only=warn)


@pytest.mark.parametrize("return_depth", [False, True], ids=["colour", "depth"])
def test_operator_backward_alerts_under_torch_deterministic_algorithms(cuda, torch_deterministic_flag, return_depth):
    from photo_slam_b200 import rasterizer
    cam, sc, act, g, c = scene_tensors(2_000, "tum", seed=1, pose_seed=2, dev=cuda, wh=(160, 120), scale_px=4.0)
    rs = rasterizer.GaussianRasterizationSettings(c["H"], c["W"], c["tanfovx"], c["tanfovy"], torch.zeros(3, device=cuda), 1.0, c["viewmatrix"],
                                                  c["projmatrix"], 3, c["campos"])

    def forward_backward():
        leaves = {k: v.clone().requires_grad_(True) for k, v in g.items()}
        means2D = torch.zeros_like(leaves["means3D"], requires_grad=True)
        out = rasterizer.GaussianRasterizer(rs)(leaves["means3D"], means2D, leaves["opacities"], shs=leaves["shs"], scales=leaves["scales"],
                                                rotations=leaves["rotations"], return_depth=return_depth)
        loss = out[0].sum() + (out[2].sum() if return_depth else 0.0)
        loss.backward()
        return leaves["means3D"].grad

    torch.use_deterministic_algorithms(False)
    assert forward_backward().abs().sum() > 0
    torch.use_deterministic_algorithms(True)
    with pytest.raises(RuntimeError, match="psb200 rasterize backward"):
        forward_backward()
    torch.use_deterministic_algorithms(True, warn_only=True)
    with pytest.warns(UserWarning, match="psb200 rasterize backward"):
        grad = forward_backward()
    assert grad.abs().sum() > 0
