"""-m gpu: the fused densify / prune / insert kernels (psb_densify_*, psb_prune_*, psb_insert_points, psb_reset_opacity) against
  (1) oracle/gs_oracle.c:orc_densify_and_prune — the reference's densifyAndPrune restated step by step in C, and
  (2) oracle/ref_densify.py — the same restated with the ATen ops the reference's LibTorch code calls, run on the GPU,
with the SAME injected normal draw. Parity: selection, compaction order and counts exact; copied rows bit-exact; computed values
(split children) to 1e-6. Reference: src/gaussian_model.cpp:193-377, 556-815."""
import math

import numpy as np
import pytest
import torch

import photo_slam_b200.synthetic as syn

pytestmark = pytest.mark.gpu


def _state(P, seed, extent, dev):
    from photo_slam_b200 import trainer
    rng = np.random.default_rng(seed)
    sc = syn.make_scene(P, syn.make_camera(160, 120, 130.0, 130.0), seed=seed)
    sc["scaling"][rng.choice(P, P // 50, replace=False)] = np.log(0.2 * extent)   # oversized: world-size prune
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    gen = torch.Generator(device=dev).manual_seed(seed)
    for t in m.exp_avg_:
        t.copy_(torch.rand(t.shape, device=dev, generator=gen) * 2 - 1)
    for t in m.exp_avg_sq_:
        t.copy_(torch.rand(t.shape, device=dev, generator=gen))
    m.xyz_gradient_accum_.copy_(torch.rand((P, 1), device=dev, generator=gen) * 0.004)
    m.denom_.fill_(2.0)
    m.denom_[::10] = 0.0
    m.xyz_gradient_accum_[::10] = 0.0                      # never seen: 0/0 -> nan -> 0
    m.max_radii2D_.copy_(torch.rand(P, device=dev, generator=gen) * 50)
    m.exist_since_iter_ = torch.arange(P, dtype=torch.int32, device=dev)
    return m


def _snapshot(m):
    c = lambda ts: [t.clone() for t in ts]
    return dict(p=c(m.tensors()), m=c(m.exp_avg_), v=c(m.exp_avg_sq_), accum=m.xyz_gradient_accum_.clone(), denom=m.denom_.clone(),
                max_radii=m.max_radii2D_.clone())


@pytest.mark.parametrize("P,max_screen_size", [(3_000, 0), (50_000, 20), (200_001, 20)])
def test_fused_densify_matches_both_oracles(cuda, P, max_screen_size):
    import oracle_c
    import ref_densify
    extent, tau, min_op = 5.0, 0.001, 0.3
    m = _state(P, 4, extent, cuda)
    st = _snapshot(m)
    exist0 = m.exist_since_iter_.clone()
    ns = m.densifySplitCount(tau, extent)
    assert ns == ref_densify.split_count(dict(st, accum=st["accum"].clone(), denom=st["denom"].clone()), tau, extent, m.percent_dense_) and ns > 10
    z = torch.randn((2 * ns, 3), device=cuda, generator=torch.Generator(device=cuda).manual_seed(9))
    # (1) C oracle on the host
    host = lambda ts: [t.cpu().numpy() for t in ts]
    op, om, ov = oracle_c.densify_and_prune(host(st["p"]), host(st["m"]), host(st["v"]), st["accum"].cpu().numpy(), st["denom"].cpu().numpy(),
                                            st["max_radii"].cpu().numpy(), tau, min_op, extent, max_screen_size, m.percent_dense_, z.cpu().numpy())
    # (2) ATen restatement on the GPU
    ref_densify.densify_and_prune(st, tau, min_op, extent, max_screen_size, m.percent_dense_, z)
    # fused kernel
    counts = m.densifyAndPrune(tau, min_op, extent, max_screen_size, samples=z)
    torch.cuda.synchronize()
    n = st["p"][0].size(0)
    assert counts[0] == n == op[0].shape[0] == m.num_points() and counts[0] == counts[1] + counts[2] + 2 * counts[3] and counts[4] == ns
    assert counts[2] > 0 and counts[3] > 0 and counts[1] < P
    names = ["xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation"]
    for name, mine, a, c in zip(names * 3, m.tensors() + m.exp_avg_ + m.exp_avg_sq_, st["p"] + st["m"] + st["v"], op + om + ov):
        assert mine.shape == a.shape, name
        assert torch.allclose(mine, a, rtol=1e-6, atol=1e-6), (name, (mine - a).abs().max().item())
        assert np.allclose(mine.cpu().numpy(), c, rtol=1e-6, atol=1e-6), name
    # copied rows are bit-exact (f_dc / f_rest / opacity / rotation are copies everywhere; moments of survivors), new rows carry zero moments
    for i in (1, 2, 3, 5):
        assert torch.equal(m.tensors()[i], st["p"][i]) and torch.equal(m.exp_avg_[i], st["m"][i]) and torch.equal(m.exp_avg_sq_[i], st["v"][i])
    K0 = counts[1]
    assert not m.exp_avg_[2][K0:].any() and not m.exp_avg_sq_[0][K0:].any()
    # statistics reset (densificationPostfix :709-711), exist_since_iter inherited from the parent row
    assert not m.xyz_gradient_accum_.any() and not m.denom_.any() and not m.max_radii2D_.any()
    assert m.xyz_gradient_accum_.shape == (n, 1) and m.max_radii2D_.shape == (n,)
    ex = m.exist_since_iter_
    assert ex.shape == (n,) and torch.equal(m.xyz_[:K0], st["p"][0][:K0])
    # a surviving original row keeps its own index as exist value (arange) and rows stay in source order within each segment
    assert (ex[:K0][1:] > ex[:K0][:-1]).all() and (ex[K0:K0 + counts[2]][1:] > ex[K0:K0 + counts[2]][:-1]).all()
    child0, child1 = ex[K0 + counts[2]:K0 + counts[2] + counts[3]], ex[K0 + counts[2] + counts[3]:]
    assert torch.equal(child0, child1)
    assert exist0.numel() == P


def test_philox_split_is_deterministic_and_standard_normal(cuda):
    extent, tau = 5.0, 0.001
    a, b, c = (_state(120_000, 6, extent, cuda) for _ in range(3))
    parents = _snapshot(a)
    ca = a.densifyAndPrune(tau, 0.0, extent, 0, seed=7, offset=3)
    cb = b.densifyAndPrune(tau, 0.0, extent, 0, seed=7, offset=3)
    cc = c.densifyAndPrune(tau, 0.0, extent, 0, seed=7, offset=4)
    assert ca == cb == cc
    assert all(torch.equal(x, y) for x, y in zip(a.tensors(), b.tensors())), "same (seed, offset) -> identical replicas"
    assert not torch.equal(a.xyz_, c.xyz_), "another offset -> another draw"
    # children of split parents: R^T (xyz_child - xyz_parent) / exp(s_parent) must be N(0, 1) per axis
    import ref_densify
    P = parents["p"][0].size(0)
    g = (parents["accum"] / parents["denom"]).nan_to_num(0.0).squeeze()
    sel = (g >= tau) & (torch.exp(parents["p"][4]).max(dim=1).values > a.percent_dense_ * extent)
    ns = int(sel.sum())
    assert ns == ca[4] == ca[3] and ns > 5000
    kids = a.xyz_[-2 * ns:]
    R = ref_densify.build_rotation(parents["p"][5][sel]).repeat(2, 1, 1)
    d = torch.bmm(R.transpose(1, 2), (kids - parents["p"][0][sel].repeat(2, 1)).unsqueeze(-1)).squeeze(-1) / torch.exp(parents["p"][4][sel]).repeat(2, 1)
    tol = 5.0 / math.sqrt(2 * ns)
    assert d.mean(dim=0).abs().max().item() < tol and (d.var(dim=0) - 1).abs().max().item() < 3 * tol, (d.mean(dim=0), d.var(dim=0))
    assert abs((d[:, 0] * d[:, 1]).mean().item()) < tol and abs((d[:ns, 0] * d[ns:, 0]).mean().item()) < tol   # axes / copies uncorrelated
    assert (d.abs() > 4.5).float().mean().item() < 1e-4 and d.abs().max().item() < 7.0


def test_prune_insert_reset_and_training_after_surgery(cuda):
    import oracle_c
    from photo_slam_b200 import trainer
    from photo_slam_b200.points import distCUDA2
    P, extent = 20_003, 5.0
    m = _state(P, 8, extent, cuda)
    st = _snapshot(m)
    ex0 = m.exist_since_iter_.clone()
    mask = torch.rand(P, device=cuda) < 0.3
    m.prunePoints(mask)
    keep = ~mask
    assert m.num_points() == int(keep.sum())
    for mine, a in zip(m.tensors() + m.exp_avg_ + m.exp_avg_sq_, st["p"] + st["m"] + st["v"]):
        assert torch.equal(mine, a[keep])
    assert torch.equal(m.xyz_gradient_accum_, st["accum"][keep]) and torch.equal(m.denom_, st["denom"][keep]) and torch.equal(m.max_radii2D_, st["max_radii"][keep])
    assert torch.equal(m.exist_since_iter_, ex0[keep])
    # insertion (increasePcd): reference gaussian_model.cpp:222-262
    n1 = m.num_points()
    before = _snapshot(m)
    pts, cols = torch.rand((301, 3), device=cuda), torch.rand((301, 3), device=cuda)
    m.increasePcd(pts, cols, iteration=77)
    assert m.num_points() == n1 + 301
    for mine, a in zip(m.tensors() + m.exp_avg_ + m.exp_avg_sq_, before["p"] + before["m"] + before["v"]):
        assert torch.equal(mine[:n1], a)
    assert torch.equal(m.xyz_[n1:], pts)
    assert torch.allclose(m.features_dc_[n1:, 0], (cols - 0.5) / 0.28209479177387814, rtol=1e-6, atol=1e-7) and not m.features_rest_[n1:].any()
    sc = torch.log(torch.sqrt(torch.clamp_min(distCUDA2(pts), 0.0000001)))
    assert torch.allclose(m.scaling_[n1:], sc.unsqueeze(1).repeat(1, 3), rtol=1e-6, atol=1e-6)
    assert torch.allclose(torch.sigmoid(m.opacity_[n1:]), torch.full((301, 1), 0.1, device=cuda), atol=1e-6)
    assert torch.equal(m.rotation_[n1:], torch.tensor([1.0, 0, 0, 0], device=cuda).repeat(301, 1))
    assert not any(t[n1:].any() for t in m.exp_avg_ + m.exp_avg_sq_) and not m.denom_.any() and m.denom_.shape == (n1 + 301, 1)
    assert (m.exist_since_iter_[n1:] == 77).all()
    # host-vector overload
    m.increasePcd([0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 1.0, 1.1, 1.2], [0.5] * 12, iteration=78)
    assert m.num_points() == n1 + 305 and m.sparse_points_xyz_.shape == (305, 3)
    # resetOpacity: values per the oracle (the reference's clamp is a no-op), opacity moments zeroed
    op = m.opacity_.clone()
    m.exp_avg_[3].fill_(1.0)
    m.resetOpacity()
    torch.cuda.synchronize()
    assert np.allclose(m.opacity_.cpu().numpy(), oracle_c.reset_opacity(op.cpu().numpy()), rtol=1e-6, atol=1e-6) and not m.exp_avg_[3].any()
    # loop-closure surface: applyScaledTransformation (xyz <- T (s xyz), log-scales * s, fresh moments)
    xyz0, sc0 = m.xyz_.clone(), m.scaling_.clone()
    T = torch.eye(4)
    T[:3, 3] = torch.tensor([0.5, -0.25, 1.0])
    m.applyScaledTransformation(1.5, T)
    assert torch.allclose(m.xyz_, xyz0 * 1.5 + T[:3, 3].to(cuda), atol=1e-5) and torch.allclose(m.scaling_, sc0 * 1.5)
    assert not m.exp_avg_[0].any() and not m.exp_avg_sq_[4].any()
    # and the model still trains after all of it
    W, H = 160, 120
    camn = syn.make_camera(W, H, 130.0, 130.0)
    c = syn.device_camera(camn, cuda)
    tr = trainer.GaussianTrainer(m)
    tr.trainForOneIteration(c, torch.rand((3, H, W), device=cuda))
    assert math.isfinite(tr.result()[0])


def test_prune_apply_without_keep_stats_zeroes_the_statistics(cuda):
    import ctypes as C
    from photo_slam_b200 import _lib, trainer

    def cm(p, m, v, accum, denom, max_radii, exist):
        c = trainer._Model()
        for i in range(6):
            c.param[i], c.exp_avg[i], c.exp_avg_sq[i] = p[i].data_ptr(), m[i].data_ptr(), v[i].data_ptr()
        c.max_radii2D, c.xyz_gradient_accum, c.denom, c.exist_since_iter = max_radii.data_ptr(), accum.data_ptr(), denom.data_ptr(), exist.data_ptr()
        return c
    m = _state(5_003, 3, 5.0, cuda)
    L, P, stream = trainer._bind(), m.num_points(), torch.cuda.current_stream().cuda_stream
    mask = torch.rand(P, device=cuda) < 0.3
    ws = torch.empty(L.psb_densify_workspace_bytes(P), dtype=torch.uint8, device=cuda)
    counts = (C.c_int * 5)()
    _lib.check(L.psb_prune_plan(P, mask.to(torch.uint8).data_ptr(), ws.data_ptr(), counts, stream), "psb_prune_plan")
    keep = ~mask
    assert counts[0] == int(keep.sum())
    d = m._blank(counts[0])
    for t in (d["accum"], d["denom"], d["max_radii"]):
        t.fill_(7.0)
    src = cm(m.tensors(), m.exp_avg_, m.exp_avg_sq_, m.xyz_gradient_accum_, m.denom_, m.max_radii2D_, m.exist_since_iter_)
    _lib.check(L.psb_prune_apply(P, C.byref(src), C.byref(cm(**d)), counts[0], ws.data_ptr(), 0, stream), "psb_prune_apply")
    torch.cuda.synchronize()
    assert not d["accum"].any() and not d["denom"].any() and not d["max_radii"].any()
    for mine, a in zip(d["p"] + d["m"] + d["v"] + [d["exist"]], m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + [m.exist_since_iter_]):
        assert torch.equal(mine, a[keep])
