"""-m gpu: the quality gate of BASELINE.json — "PSNR within 0.1 dB of reference after equal iterations" — on a run that exercises the whole
trainer surface: 600 iterations over 6 keyframes of a 200 k-Gaussian scene at 640x480, with densification (clone / split / prune every
100 iterations) and the SH-degree schedule, psb200 (fused step + fused densify) vs the reference chain (oracle/ref_trainer.py: the
reference's own rasterizer kernels + ATen ops + ATen densification restated from src/gaussian_model.cpp:556-815). The reference run's
PSNR, densification counts and Gaussian count are stored in tests/golden/test_quality_gpu.npz (written on an H100 by
tests/golden/make_ref_golden.py from reference_cases() below)."""
import math

import numpy as np
import pytest
import torch

import photo_slam_b200.synthetic as syn
from helpers import Gold

pytestmark = pytest.mark.gpu
LRS = [0.00016, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]
MODULE = "test_quality_gpu"


def _run(cuda, gold=None):
    """psb200's 600 iterations; with gold=None the reference chain runs beside it and its record is returned, otherwise the
    reference's stored densification threshold and split counts drive the same schedule."""
    from photo_slam_b200 import trainer
    gt_scene, cams = syn.quality_scene()
    views = [syn.device_camera(cam, cuda) for cam in cams]
    gt_model = trainer.GaussianModel.from_numpy(gt_scene, cuda)
    gt_tr = trainer.GaussianTrainer(gt_model)
    gts = [gt_tr.render(c).clamp(0, 1).clone() for c in views]
    # the trainee: a perturbed, thinned copy of the scene (so densification has something to do)
    start = syn.thinned_trainee(gt_scene)
    n0 = len(start["xyz"])

    opt = trainer.GaussianOptimizationParams()
    model = trainer.GaussianModel.from_numpy(start, cuda)
    model.trainingSetup(opt)
    model.lr_ = list(LRS)
    model.setShDegree(0)
    tr = trainer.GaussianTrainer(model, opt)
    if gold is None:
        import ref_trainer
        ref = ref_trainer.RefTrainer(start, cuda, LRS, sh_degree=0)

    def psnr_of(render):
        return float(np.mean([10.0 * math.log10(1.0 / ((render(c) - g) ** 2).mean().item()) for c, g in zip(views, gts)]))

    p_start = psnr_of(lambda c: tr.render(c))
    extent, min_op, tau = 1.0, 0.005, None     # percent_dense * extent = 0.01: the scene's scales straddle it, so both clone and split fire
    if gold is not None:
        tau = gold["tau"]
    gen = torch.Generator(device=cuda).manual_seed(5)
    counts, ns_refs = [], []
    for it in range(1, 601):
        c, g = views[it % 6], gts[it % 6]
        if it % 150 == 0:                                   # SH degree schedule (oneUpShDegree, gaussian_mapper.cpp:672-674)
            model.oneUpShDegree()
            if gold is None:
                ref.sh_degree = model.active_sh_degree_
        tr.trainForOneIteration(c, g)
        tr.result()
        if gold is None:
            ref.train_for_one_iteration(c, g)
        if it % 100 == 0 and it <= 500:
            if tau is None:                                 # one threshold for both sides and all rounds: top 5 % of the mean screen gradients
                grads = (model.xyz_gradient_accum_ / model.denom_).nan_to_num(0.0).squeeze()
                tau = float(torch.quantile(grads[grads > 0][:1_000_000], 0.95))
            if gold is None:
                ns_ref = __import__("ref_densify").split_count(dict(p=[t.detach() for t in ref.tensors()], accum=ref.xyz_gradient_accum.clone(),
                                                                     denom=ref.denom.clone()), tau, extent, 0.01)
            else:
                ns_ref = int(gold.full("ns_ref")[len(ns_refs)])
            ns_refs.append(ns_ref)
            z = torch.randn((2 * max(ns_ref, model.densifySplitCount(tau, extent)), 3), device=cuda, generator=gen)
            cm = model.densifyAndPrune(tau, min_op, extent, 20, samples=z[:2 * model.densifySplitCount(tau, extent)])
            if gold is None:
                ref.densify_and_prune(tau, min_op, extent, 20, 0.01, z[:2 * ns_ref])
            counts.append((it, cm, ref.xyz.size(0) if gold is None else int(gold.full("p_new")[len(counts)])))
    torch.cuda.synchronize()
    if gold is None:
        return dict(tau=tau, ns_ref=np.array(ns_refs), p_new=np.array([nr for _, _, nr in counts]), psnr=psnr_of(lambda c: ref.render(c)[0].detach()),
                    psnr_start=p_start, points=ref.xyz.size(0))
    p_psb = psnr_of(lambda c: tr.render(c))
    p_ref, n_ref = gold["psnr"], gold["points"]
    print(f"PSNR over 6 views: start {p_start:.3f} dB -> psb200 {p_psb:.3f} dB, reference {p_ref:.3f} dB; Gaussians {n0} -> psb {model.num_points()} / ref {n_ref}")
    for it, cm, nr in counts:
        print(f"  densify @{it}: psb (P_new, kept, clones, children/copy, split) = {cm}; reference P_new = {nr}")
    assert sum(cm[2] for _, cm, _ in counts) > 100 and sum(cm[3] for _, cm, _ in counts) > 100, "the run must exercise both clone and split"
    assert p_psb > p_start + 2.0 and p_ref > gold["psnr_start"] + 2.0, "training must improve the picture"
    assert abs(p_psb - p_ref) < 0.1, (p_psb, p_ref)
    assert abs(model.num_points() - n_ref) <= 0.02 * n_ref


def test_psnr_within_a_tenth_of_a_db_after_600_iterations_with_densification(cuda):
    _run(cuda, Gold(MODULE, "run"))


def reference_cases(cuda):
    """(case, {name: array | scalar}) of the reference chain's run (tests/golden/make_ref_golden.py)."""
    yield "run", _run(cuda)
