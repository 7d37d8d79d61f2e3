"""-m gpu: the normal, depth-normal consistency and distortion terms on the data-parallel paths — the NVLink step (psb_dp_step_dist),
the slab pipeline (psb_trainer_backward_begin_dist -> psb_trainer_backward_slab) and the flat split path (psb_trainer_backward_dist) —
on a DataParallelTrainer(geometry_terms=True), against the fused step with the same terms on one GPU, and ranks with different terms in
one step (one per GPU when the box has >= 2, four processes sharing the GPU otherwise) against the 1-rank step on the summed gradients."""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

import shared_device
from test_dist_gpu import _dist_planes32
from test_dp_depth_gpu import LRS, SLABS, _assert_same_state, _finish, _inputs, _model, _render_target
from test_normal_gpu import _grad_of_l1, _same, _settled, _state, _targets

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAMBDA_DEPTH, LAMBDA_NORMAL, LAMBDA_DN, LAMBDA_DIST = 0.1, 0.05, 0.05, 0.1
ALPHA_MIN, JUMP = 0.5, 0.05


def _scene(cuda, P=12_345):
    """test_dp_depth_gpu's scene, view, colour and depth targets, and a normal target: the sensor normals of the model's own rendered
    depth x 1.02"""
    from photo_slam_b200 import trainer
    sc, c, gt, gd = _inputs(cuda, P)
    tr = trainer.GaussianTrainer(_model(sc, cuda))
    D = torch.empty((c["H"], c["W"]), device=cuda)
    tr.render(c, out_depth=D)
    gn = trainer.normals_from_depth(c, (D * 1.02).contiguous())
    torch.cuda.synchronize()
    assert (gn != 0).any(0).sum().item() > 1000
    return sc, c, gt, gd, gn


def _terms(name, gd, gn):
    n = dict(gt_normal=gn, lambda_normal=LAMBDA_NORMAL)
    dn = dict(lambda_dn=LAMBDA_DN, dn_alpha_min=ALPHA_MIN, dn_max_rel_jump=JUMP)
    return {"plain": {}, "normal": n, "normal_dn": dict(n, **dn), "dist": dict(lambda_dist=LAMBDA_DIST),
            "all": dict(n, **dn, gt_depth=gd, lambda_depth=LAMBDA_DEPTH, lambda_dist=LAMBDA_DIST)}[name]


def _has(name):
    """which of depth_l1, normal_l1, dn, dist the terms `name` report as non-zero"""
    return {"plain": (0, 0, 0, 0), "normal": (0, 1, 0, 0), "normal_dn": (0, 1, 1, 0), "dist": (0, 0, 0, 1), "all": (1, 1, 1, 1)}[name]


def _assert_same_result(ra, rb, what=""):
    """test_dp_depth_gpu's _assert_same_result over the seven terms of result_dist()"""
    assert abs(ra[0] - rb[0]) <= 2e-5 * max(1.0, abs(ra[0])), (what, ra, rb)
    for k in range(3, 7):
        assert abs(ra[k] - rb[k]) <= 1e-5 * max(1.0, abs(ra[k])), (what, k, ra, rb)


def _check_terms(r, name):
    for k, on in zip(range(3, 7), _has(name)):
        assert (r[k] != 0.0) == bool(on), (name, r)


@pytest.mark.parametrize("aa", [False, True], ids=["plain", "aa"])
@pytest.mark.parametrize("name", ["normal", "normal_dn", "dist", "all"])
def test_p2p_terms_world1_equal_fused_steps(cuda, name, aa):
    from photo_slam_b200 import trainer
    sc, c, gt, gd, gn = _scene(cuda)
    a, b = _model(sc, cuda), _model(sc, cuda)
    ta, tb = trainer.GaussianTrainer(a, antialiasing=aa), trainer.DataParallelTrainer(b, mode="p2p", antialiasing=aa, geometry_terms=True)
    assert tb.mode == "p2p"
    kw = _terms(name, gd, gn)
    for it in range(4):
        ta.trainForOneIteration(c, gt, **kw)
        tb.trainForOneIteration(c, gt, **kw)
        ra, rb = ta.result_dist(), tb.result_dist()
        _check_terms(ra, name)
        _assert_same_result(ra, rb, it)
    _finish(tb)
    assert tb.status() == 0
    _assert_same_state(a, b, name)
    tb.close()


def test_slab_pipeline_and_flat_path_with_all_terms_equal_fused_steps(cuda):
    from photo_slam_b200 import trainer
    sc, c, gt, gd, gn = _scene(cuda)
    models = [_model(sc, cuda) for _ in range(3)]
    trs = [trainer.DataParallelTrainer(models[0], **SLABS, geometry_terms=True),
           trainer.DataParallelTrainer(models[1], mode="nccl", pipeline=False, geometry_terms=True), trainer.GaussianTrainer(models[2])]
    assert trs[0].pipeline and not trs[1].pipeline
    kw = _terms("all", gd, gn)
    for it in range(3):
        res = []
        for tr in trs:
            tr.trainForOneIteration(c, gt, **kw)
            res.append(tr.result_dist())
        _check_terms(res[0], "all")
        _assert_same_result(res[0], res[1], ("flat", it))
        _assert_same_result(res[0], res[2], ("fused", it))
    torch.cuda.synchronize()
    _assert_same_state(models[0], models[1], "flat")
    _assert_same_state(models[2], models[0], "fused")


@pytest.mark.parametrize("masked", [False, True], ids=["nomask", "mask"])
def test_gradient_mode_equals_the_split_path_bit_for_bit(cuda, masked):
    """psb_trainer_backward_dist's raw gradients against DataParallelTrainer.render(out_normal, out_depth2) + the terms' pixel gradients
    formed as test_dist_gpu forms them + DataParallelTrainer.backwardPixels(..., grads=), in deterministic mode"""
    from photo_slam_b200 import _lib, trainer
    from photo_slam_b200.parallel import GradBuffer
    cam, sc = _settled("b")
    import photo_slam_b200.synthetic as syn
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    gt, mask, gd, gn = _targets(H, W, cuda)
    msk = mask if masked else None
    m = _model(sc, cuda)
    tr = trainer.DataParallelTrainer(m, mode="nccl", pipeline=False, deterministic=True, geometry_terms=True)
    tr._apply_deterministic()
    tr.opt.lambda_dssim = 0.2
    P = m.num_points()
    # built-in loss, gradient mode
    kern = GradBuffer(P, cuda)
    cm, cc, cs = m._cmodel(), trainer._ccamera(c), tr._cstep(True)
    d = trainer._Depth(gd.data_ptr(), LAMBDA_DEPTH, None)
    nrm = trainer._Normal(gn.data_ptr(), LAMBDA_NORMAL, None)
    dn = trainer._Dn(LAMBDA_DN, ALPHA_MIN, JUMP, None)
    ds = trainer._Dist(LAMBDA_DIST, None)
    ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in kern.segments])
    img_k = torch.empty((3, H, W), device=cuda)
    _lib.check(tr.L.psb_trainer_backward_dist(*tr._call_args(m, cm, cc, cs, gt, msk, img_k, None), ptrs, C.byref(d), None, None, C.byref(nrm),
                                              C.byref(dn), C.byref(ds), torch.cuda.current_stream().cuda_stream), "psb_trainer_backward_dist")
    res = tr.result_dist()
    assert all(x > 0 for x in res[3:7]), res
    torch.cuda.synchronize()
    # the split path
    img, D, A, N, M = (torch.empty((3, H, W), device=cuda), torch.empty((H, W), device=cuda), torch.empty((H, W), device=cuda),
                       torch.empty((3, H, W), device=cuda), torch.empty((H, W), device=cuda))
    tr.render(c, img, out_depth=D, out_alpha=A, out_normal=N, out_depth2=M)
    _, _, _, g = trainer.fused_loss(img, gt, msk, 0.2)
    valid = msk[0] != 0 if msk is not None else torch.ones((H, W), dtype=torch.bool, device=cuda)
    vd, vn = (gd > 0) & valid, (gn != 0).any(0) & valid
    grads = (_grad_of_l1(D, gd, vd, LAMBDA_DEPTH), torch.zeros_like(A), _grad_of_l1(N, gn, vn, LAMBDA_NORMAL))
    _, _, grads = trainer._dn_loss(c, D, A, N, msk[0].contiguous() if msk is not None else None, LAMBDA_DN, ALPHA_MIN, JUMP, grads=grads)
    gD, gA, gN = grads
    gD, gA, gM = _dist_planes32(D, A, M, valid, LAMBDA_DIST, gD, gA)
    split = GradBuffer(P, cuda)
    tr.backwardPixels(g, gD, gA, grads=split.views(), dL_dnormal=gN, dL_ddepth2=gM)
    tr.result()
    torch.cuda.synchronize()
    assert torch.equal(img, img_k)
    for name, x, y in zip(trainer.GROUPS, kern.views(), split.views()):
        assert x.abs().sum().item() > 0, name
        assert torch.equal(x, y), (name, (x - y).abs().max().item())


class _Route:
    """the library with psb_dp_step_dist and psb_trainer_backward_begin_dist routed to psb_dp_step_depth and
    psb_trainer_backward_begin_depth (which the three term records, all NULL, are dropped for)"""

    def __init__(self, L):
        self._L = L

    def __getattr__(self, n):
        return getattr(self._L, n)

    def psb_dp_step_dist(self, *a):
        assert a[-4:-1] == (None, None, None)
        return self._L.psb_dp_step_depth(*a[:-4], a[-1])

    def psb_trainer_backward_begin_dist(self, *a):
        assert a[-4:-1] == (None, None, None)
        return self._L.psb_trainer_backward_begin_depth(*a[:-4], a[-1])


@pytest.mark.parametrize("kw", [dict(mode="p2p"), SLABS], ids=["p2p", "slabs"])
def test_null_terms_are_the_depth_calls_bit_for_bit(cuda, kw):
    from photo_slam_b200 import trainer
    sc, c, gt, gd, gn = _scene(cuda)
    states = []
    for route in (False, True):
        m = _model(sc, cuda)
        tr = trainer.DataParallelTrainer(m, deterministic=True, **kw, geometry_terms=True)
        if route:
            tr.L = _Route(tr.L)
        res = []
        for it in range(3):
            tr.trainForOneIteration(c, gt, **(dict(gt_depth=gd, lambda_depth=LAMBDA_DEPTH) if it != 1 else {}))
            res.append(tr.result_depth())
        _finish(tr)
        states.append((repr(res), _state(m)))
        if hasattr(tr, "close"):
            tr.close()
    assert states[0][0] == states[1][0]
    assert _same(states[0][1], states[1][1])


@pytest.mark.parametrize("name,group", [("normal", 5), ("dist", 0)])
def test_p2p_rows_reached_only_by_the_terms_are_updated_like_the_fused_step(cuda, name, group):
    """Every colour target equals the render and lambda_dssim = 0: only the term reaches the rows. A normal-only step moves rotations,
    a distortion-only step positions, of more than 100 rows, and the same rows as the fused step."""
    from photo_slam_b200 import trainer
    sc, c, gt, gd, gn = _scene(cuda, 20_000)
    a, b = _model(sc, cuda), _model(sc, cuda)
    ta, tb = trainer.GaussianTrainer(a), trainer.DataParallelTrainer(b, mode="p2p", geometry_terms=True)
    before = a.tensors()[group].clone()
    for tr in (ta, tb):
        tr.opt.lambda_dssim = 0.0
        tr.trainForOneIteration(c, _render_target(tr, c), **_terms(name, gd, gn))
    ra, rb = ta.result_dist(), tb.result_dist()
    _finish(tb)
    assert ra[1] == 0.0 and rb[1] == 0.0
    _check_terms(rb, name)
    _assert_same_result(ra, rb)
    pa, pb = a.tensors()[group], b.tensors()[group]
    moved_a, moved_b = (pa != before).any(dim=1), (pb != before).any(dim=1)
    assert moved_b.sum().item() > 100, moved_b.sum().item()
    assert (moved_a != moved_b).sum().item() <= 2e-3 * moved_a.numel()
    rows = moved_a & moved_b
    frac = ((pa[rows] - pb[rows]).abs() > 0.5 * LRS[group]).float().mean().item()
    assert frac < 2e-3, frac
    _assert_same_state(a, b)
    tb.close()


@pytest.mark.parametrize("kw", [dict(mode="p2p"), SLABS], ids=["p2p", "slabs"])
def test_term_and_plain_steps_alternate_like_fused_steps(cuda, kw):
    """normal, plain, dist, plain, all, plain, normal+dn with every colour target equal to the render: 16-float and 12-float sink rows
    and dL/dz alternate, and each step reaches its rows through its terms alone. A per-Gaussian kernel that read a row of the other
    width, or left a gradient in the sink, would lose it from its own step and add it to a later one; the sequence must equal the same
    sequence of fused steps."""
    from photo_slam_b200 import trainer
    sc, c, gt, gd, gn = _scene(cuda)
    a, b = _model(sc, cuda), _model(sc, cuda)
    ta, tb = trainer.GaussianTrainer(a), trainer.DataParallelTrainer(b, **kw, geometry_terms=True)
    for tr in (ta, tb):
        tr.opt.lambda_dssim = 0.0
    for it, name in enumerate(("normal", "plain", "dist", "plain", "all", "plain", "normal_dn")):
        res = []
        for tr in (ta, tb):
            tr.trainForOneIteration(c, _render_target(tr, c), **_terms(name, gd, gn))
            res.append(tr.result_dist())
        assert res[0][1] == 0.0 and res[1][1] == 0.0, "the colour target must equal the render"
        _check_terms(res[1], name)
        _assert_same_result(res[0], res[1], (it, name))
    _finish(tb)
    _assert_same_state(a, b)
    tb.close()


def test_p2p_terms_bit_identical_run_to_run(cuda):
    from photo_slam_b200 import trainer
    sc, c, gt, gd, gn = _scene(cuda)
    runs = []
    for _ in range(2):
        m = _model(sc, cuda)
        tr = trainer.DataParallelTrainer(m, mode="p2p", deterministic=True, geometry_terms=True)
        res = []
        for it in range(20):
            tr.trainForOneIteration(c, gt, **_terms("all", gd, gn))
            res.append(tr.result_dist())
        _finish(tr)
        runs.append((repr(res), _state(m)))
        tr.close()
    assert runs[0][0] == runs[1][0]
    assert _same(runs[0][1], runs[1][1])


@pytest.mark.parametrize("kw", [dict(mode="p2p"), SLABS], ids=["p2p", "slabs"])
def test_overflowing_view_with_the_terms_is_dropped_not_retried(cuda, kw):
    """test_overflowing_depth_view_is_dropped_not_retried with every term: the view contributes a zero gradient, result_dist() is all NaN,
    and the next step of the same view trains."""
    from helpers import scene_tensors
    from photo_slam_b200 import trainer
    P, wh = 2_000, (640, 480)
    cam, sc, act, g, c = scene_tensors(P, "tum", seed=2, pose_seed=None, dev=cuda, wh=wh, scale_px=150.0)
    gt, _, gd, gn = _targets(wh[1], wh[0], cuda)
    m = _model(sc, cuda)
    tr = trainer.DataParallelTrainer(m, **kw, geometry_terms=True)
    before = [t.clone() for t in m.tensors()]
    kwt = _terms("all", gd, gn)
    tr.trainForOneIteration(c, gt, **kwt)
    res = tr.result_dist()
    _finish(tr)
    assert res[7] > 6 * P + 65536 and tr.dropped_views == 1
    assert all(x != x for x in res[:7]), res
    for x, y in zip(before, m.tensors()):
        assert torch.equal(x, y), "a dropped view must not move the parameters (zero gradient, zero moments)"
    assert not any(t.any() for t in m.exp_avg_ + m.exp_avg_sq_)
    tr.trainForOneIteration(c, gt, **kwt)
    res2 = tr.result_dist()
    _finish(tr)
    assert res2[0] == res2[0] and res2[4] > 0.0 and res2[6] > 0.0 and tr.dropped_views == 1
    assert not torch.equal(before[0], m.xyz_) and not torch.equal(before[5], m.tensors()[5])
    tr.close()


def test_slab_after_a_begin_that_failed_before_its_normal_pass_is_refused(cuda):
    """_begin_dist records 16-float rows before its pass; when it fails before the pass made them, a _slab must not read them"""
    from photo_slam_b200 import trainer
    sc, c, gt, gd, gn = _scene(cuda)
    m = _model(sc, cuda)
    tr = trainer.DataParallelTrainer(m, **SLABS, geometry_terms=True)
    tr.trainForOneIteration(c, gt)
    tr.result()
    torch.cuda.synchronize()
    P = m.num_points()
    cm, cc, cs = m._cmodel(), trainer._ccamera(c), tr._cstep(True)
    nrm = trainer._Normal(gn.data_ptr(), LAMBDA_NORMAL, None)
    args = tr._call_args(m, cm, cc, cs, gt, None, None, None)
    args = (*args[:6], None, *args[7:])           # no colour target: the call fails after it recorded the mode
    stream = torch.cuda.current_stream().cuda_stream
    assert tr.L.psb_trainer_backward_begin_dist(*args, None, C.byref(nrm), None, None, stream) == -1
    first, count = tr.grads.slabs[0]
    ptrs = (C.c_void_p * 6)(*tr.grads.kernel_pointers(0))
    assert tr.L.psb_trainer_backward_slab(tr.h, P, 16, C.byref(cm), C.byref(cc), C.byref(cs), first, count, ptrs, stream) == -1
    assert b"no matching backward_begin" in tr.L.psb_last_error()
    tr.trainForOneIteration(c, gt, **_terms("normal", gd, gn))
    r = tr.result_dist()
    torch.cuda.synchronize()
    assert r[4] > 0.0, r


def _launch(world, mode, P, steps=3, timeout=420):
    port = 29500 + ((os.getpid() + 300) % 400)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "dp_terms_worker.py"), mode, str(P), str(steps)]
    env = dict(os.environ, PSB_DP_TIMEOUT_MS="15000")
    return subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_multi_rank_mixed_terms_replicas_identical_and_equal_summed_gradient_step(cuda, mode):
    """Ranks train with normal+dn, dist, no term and all terms in turn (mode="nccl" runs the slab pipeline at world > 1). On a single GPU,
    p2p runs four ranks sharing it (tests/shared_device.py), one for each set of terms."""
    n = torch.cuda.device_count()
    if n < 2:
        if mode != "p2p":
            pytest.skip("NCCL needs one GPU per rank: >= 2 GPUs")
        why = shared_device.unavailable()
        if why:
            pytest.skip(why)
        codes, out, tails = shared_device.launch(os.path.join(ROOT, "tests", "dp_terms_worker.py"), [mode, 30_001, 3], 4, timeout=600)
        assert codes == [0] * 4 and "DP_TERMS_WORKER_OK" in out, tails
        print(out.strip().splitlines()[-1])
        return
    world = 2 if n < 4 else (4 if n < 8 else 8)
    r = _launch(world, mode, 30_001)
    assert r.returncode == 0 and "DP_TERMS_WORKER_OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
    print(r.stdout.strip().splitlines()[-1])
