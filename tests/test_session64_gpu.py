"""-m gpu: training across row surgery against the float64 session truth of tests/session64.py. A Photo-SLAM mapper densifies, prunes,
inserts, seeds, relocates and grows the map between steps, resets opacities, applies loop-closure transforms, recomputes the 3D filter,
raises the SH degree and moves the learning rates. Each of those leaves per-row state (the trainer context's sink, seed rows and
deterministic slots, adam_live_, filter_3D_, the exposure rows, the data-parallel arena or gradient buffer) that the next fused step reads.

A GaussianTrainer session (SESSIONS: flag set, deterministic mode, scene of test_step64_gpu) runs, with updateLearningRate(step) before
every step but one and a compared step after every event: densifyAndPrune (P grows), a step with the consistency term, prunePoints of
~30 % (P falls below its pre-densify value, across multiples of 128, to 1 or 3 mod 4), a step with the distortion term, increasePcd of 301
points (P grows back into freed capacity; new rows reached for the first time), every set*LearningRate (the xyz one held for the next step)
with setShDegree(3), a render, resetOpacity, applyScaledTransformation, backwardPixels(grads=...), seedFromDepth and, with reg,
relocateGaussians then addNewGaussians with injected uniforms (the pair mcmcRefine runs); computeFilter3D after every surgery with f3d.
Every compared step is anchored (the truth steps the state read from the kernels' model) and compared with test_step64_gpu's gates; the
learning rates, the SH degree and the 3D filter in force are the truth's own. At every surgery, copied rows are checked bit for bit,
computed rows against the restatement with the per-operation tests' tolerances, and new rows for zero moments; the next step checks the
adam_live contract.

A DataParallelTrainer session at world 1 (p2p, the flat nccl path and the slab pipeline, each with and without depth, deterministic):
steps, gather_moments() and sync_densify_stats(), densifyAndPrune, a step without rebuild() (refused with ValueError, the model and the
iteration untouched), rebuild(), compared steps, prunePoints, rebuild(), a step, a second densify, rebuild() and a step at D = 3.

Gates: test_step64_gpu's, along a trajectory (GATE_STEP_TRAJ). The largest values measured on an H100 80GB HBM3 (700 W power limit) over all
sessions sit in the comments below. The whole file ran in 1.5 minutes there.
"""
import math

import numpy as np
import pytest
import torch

import filter3d64 as f3d64
import photo_slam_b200.synthetic as syn
import seed64
import session64
import step64
from test_filter3d_gpu import _packed
from test_mcmc_gpu import _compare as _compare_mcmc, _host, _safe_uniforms, _w32
from test_step64_gpu import (BG, GATE_LOSS, GATE_MOM, GATE_STEP_TRAJ, H, LAMBDA_DEPTH, SCENES, W, _assert_gates, _cams, _compare,
                             TINY, _first_moments, _kernel_step, _model, _relnorm, _settled_state, _step_err, _targets, _targets64,
                             _trainer)

pytestmark = pytest.mark.gpu

MIN_OP = 0.005

# test_step64_gpu's gates; the largest values measured over all sessions here (H100 80GB HBM3, 700 W power limit):
#   loss scalars (GATE_LOSS 1e-5): 3.6e-6 (ssim)
#   parameter step (GATE_STEP_TRAJ 1e-4, in lr): 9.1e-5 (rotation, p2p at world 1). Every value above 5e-5 (the NEAR-GATE lines) was an
#     element that step64's exclusion rule names ill-conditioned (|g| and sqrt(v) below TINY max|g|; measured |g| / max|g| <= 1e-5): Adam
#     normalises its float32 noise. Such an element either stays below the gate or is excluded and counted against GATE_EXCLUDED, so it
#     cannot fail the step gate
#   moments (GATE_MOM 4e-5): 1.4e-5 (xyz second moment)
#   xyz_gradient_accum (GATE_ACCUM 1e-5): 2.0e-6
TOL_FILTER = 1e-6         # the 3D filter against filter3d64, relative to the value plus the rounding scale of its depth: measured 9.3e-8


def _opt(fl):
    """a schedule short enough that the xyz learning rate moves by ~8 % per step"""
    from photo_slam_b200 import trainer
    return trainer.GaussianOptimizationParams(position_lr_init=3.2e-4, position_lr_final=3.2e-5, position_lr_max_steps=30, mcmc=fl.reg,
                                              mcmc_noise_lr=0.0)


def _rows(m):
    d = lambda t: t.detach().double().clone()
    return dict(p=[d(t) for t in m.tensors()], m=[d(t) for t in m.exp_avg_], v=[d(t) for t in m.exp_avg_sq_], accum=d(m.xyz_gradient_accum_),
                denom=d(m.denom_), max_radii=d(m.max_radii2D_))


def _gap(vals, q):
    """a threshold near quantile q of vals that lies at least 1e-4 (relative) from every value"""
    v = np.unique(np.asarray(vals, np.float64))
    i = int(q * (len(v) - 1))
    for j in list(range(i, len(v) - 1)) + list(range(i - 1, -1, -1)):
        if v[j + 1] - v[j] > 2e-4 * v[j + 1]:
            return 0.5 * (v[j] + v[j + 1])
    raise AssertionError("no gap")


class Run:
    """one session on one model: the kernels' model m and trainer tr, the truth's Session, and the checks"""

    def __init__(self, cuda, fl, det, scene, conv=session64.SESSION_CONV, dp=None):
        from photo_slam_b200 import trainer
        self.dev, self.fl, self.det = cuda, fl, det
        self.cams = _cams()
        self.tg = _targets(cuda)
        self.tg64 = _targets64(self.tg, BG)
        self.opt = _opt(fl)
        m = _model(SCENES[scene](), cuda, fl, self.cams)
        m.trainingSetup(self.opt)
        m.setShDegree(2)
        self.m = m
        self.ses = session64.Session(self.opt, 2, conv)
        if fl.f3d:
            self.ses.set_filter(m.filter_3D_.double().clone())
        if dp is None:
            _first_moments(m, fl, self.cams[0], self.tg64)
            self.tr = _trainer(m, fl, det)
        else:
            st, cam64, _ = _settled_state(m, fl, self.cams[1], self.tg64, 31)
            st["E"] = None
            from test_step64_gpu import _seed_moments
            _seed_moments(m, step64.grads64(st, cam64, self.tg64, fl)["grads"], None)
            self.tr = trainer.DataParallelTrainer(m, background=torch.tensor(BG, device=cuda), **dp)
            self.tr.render(syn.device_camera(self.cams[1], cuda))
        self.dp = dp
        self.n = 0
        self.worst, self.excl = {}, {}
        self.sizes = [m.num_points()]
        self.d3 = False
        self.splits = 0

    def cam(self, i=None):
        return self.cams[(self.n if i is None else i) % 3]

    def c(self, i=None):
        return syn.device_camera(self.cam(i), self.dev)

    def _note(self, errs):
        for q, v in errs.items():
            self.worst[q] = max(self.worst.get(q, 0.0), v)

    # ---- a compared step ----------------------------------------------------------------------------------------------------------
    def step(self, schedule=True):
        """one anchored, compared step; schedule=False: the xyz learning rate stays as a setter left it"""
        m, fl = self.m, self.fl
        if schedule:
            m.updateLearningRate(m.step_)
            self.ses.update_lr(m.step_)
        e = None if self.dp is not None else self.n % 2
        st, cam64, mg = _settled_state(m, fl, self.cam(), self.tg64, 1000 + self.n, e or 0)
        if self.dp is not None:
            st["E"] = None
            c = self.c()
            self.tr.trainForOneIteration(c, self.tg["gt"], self.tg["mask"], gt_depth=self.tg["depth"] if fl.depth else None,
                                         lambda_depth=LAMBDA_DEPTH if fl.depth else 0.0)
            loss = self.tr.result_depth()[:4]
            if self.tr.mode == "p2p":
                self.tr.sync()
            torch.cuda.synchronize()
            assert self.tr.dropped_views == 0 and self.tr.status() == 0
        else:
            loss = _kernel_step(self.tr, m, self.c(), self.tg, fl, e)
        before = self.ses.state(st)
        r = self.ses.step(st, cam64, self.tg64, fl)
        errs, ex, _ = _compare(m, before, r, fl, loss, live=self.dp is None, exposure_id=e, step_gate=GATE_STEP_TRAJ)
        self._note(errs)
        self._near_gate(before, r, errs)
        for q, v in ex.items():
            self.excl[q] = self.excl.get(q, 0) + v
        self.d3 |= before["D"] == 3
        self.n += 1
        self.sizes.append(m.num_points())
        return errs

    def _near_gate(self, before, r, errs):
        """prints the element behind a step error above half the gate: its gradient against the group's, its moments before the step"""
        m = self.m
        P = m.num_points()
        for i, k in enumerate(step64.GROUPS):
            if errs[f"step-{k}"] <= 0.5 * GATE_STEP_TRAJ:
                continue
            p1, ref, g = m.tensors()[i].detach().double(), r["state"]["params"][k], r["grads"][k]
            gmax = float(g.abs().max())
            ulp = (torch.nextafter(p1.float(), torch.full_like(p1.float(), math.inf)).double() - p1).abs()
            e = ((p1 - ref).abs() - ulp).clamp_min(0) / before["lr"][i]
            ill = (g.abs() < TINY * gmax) & (before["v"][k].sqrt() < TINY * gmax)
            e[ill & (e > GATE_STEP_TRAJ)] = 0.0          # excluded and counted by _compare
            j = int(e.reshape(-1).argmax())
            row = j // (g.numel() // P)
            f_ = lambda t: float(t.reshape(-1)[j])
            fresh = all(not before[q][k][row].any() for q in ("m", "v"))
            print(f"NEAR-GATE {k} err={f_(e):.2e} row={row} |g|/gmax={abs(f_(g)) / gmax:.2e} m0={f_(before['m'][k]):.2e} "
                  f"sqrt(v0)/gmax={math.sqrt(f_(before['v'][k])) / gmax:.2e} ill={bool(ill.reshape(-1)[j])} zero-moment row={fresh}")

    # ---- uncompared calls ---------------------------------------------------------------------------------------------------------
    def dn_step(self):
        self.tr.trainForOneIteration(self.c(), self.tg["gt"], self.tg["mask"], lambda_dn=0.05, exposure_id=1)
        self.tr.result_dn()

    def dist_step(self):
        self.tr.trainForOneIteration(self.c(), self.tg["gt"], self.tg["mask"], lambda_dist=0.1, gt_depth=self.tg["depth"], lambda_depth=LAMBDA_DEPTH)
        self.tr.result_dist()

    def render(self):
        self.tr.render(self.c(), out_depth=torch.empty((H, W), device=self.dev))

    def backward_pixels(self):
        self.tr.render(self.c())
        gen = torch.Generator(device=self.dev).manual_seed(self.n)
        grads = [torch.zeros_like(t) for t in self.m.tensors()]
        self.tr.backwardPixels(1e-3 * torch.randn((3, H, W), device=self.dev, generator=gen), grads=grads)
        self.tr.result()

    # ---- surgeries ----------------------------------------------------------------------------------------------------------------
    def check_rows(self, want, approx=None, new=None):
        """the model's rows against the truth's row state: groups in approx (q -> (rows [P] bool, rtol, atol)) to tolerance on those rows,
        every other element bit for bit; moments -> 'mom' errors (bit for bit: 0); new rows carry zero moments"""
        m, approx = self.m, approx or {}
        P = m.num_points()
        assert want["p"][0].shape[0] == P, (want["p"][0].shape[0], P)
        errs = {}
        for q, (k, t) in enumerate(zip(step64.GROUPS, m.tensors())):
            a, b = t.detach().double(), want["p"][q]
            rows = approx[q][0] if q in approx else torch.zeros(P, dtype=torch.bool, device=self.dev)
            assert torch.equal(a[~rows], b[~rows]), f"{k}: a copied row differs"
            if rows.any():
                rtol, atol = approx[q][1:]
                atol = atol[rows] if torch.is_tensor(atol) else atol
                d = (a[rows] - b[rows]).abs() - rtol * b[rows].abs() - atol
                assert float(d.max()) <= 0.0, (k, float(d.max()))
            errs[f"mom-m-{k}"] = _relnorm(m.exp_avg_[q], want["m"][q])
            errs[f"mom-v-{k}"] = _relnorm(m.exp_avg_sq_[q], want["v"][q])
            if new is not None:
                assert not m.exp_avg_[q][new].any() and not m.exp_avg_sq_[q][new].any(), f"{k}: a new row has moments"
        for k in ("accum", "denom", "max_radii"):
            assert torch.equal(getattr(m, {"accum": "xyz_gradient_accum_", "denom": "denom_", "max_radii": "max_radii2D_"}[k]).double().reshape(-1),
                               want[k].double().reshape(-1)), k
        return errs

    def exact(self, errs):
        assert all(v == 0.0 for k, v in errs.items() if k.startswith("mom")), errs

    def filter3d(self):
        """computeFilter3D on the three cameras against filter3d64; the truth then puts it in force"""
        if not self.fl.f3d:
            return
        m = self.m
        dc = [syn.device_camera(c, self.dev) for c in self.cams]
        m.computeFilter3D(dc)
        torch.cuda.synchronize()
        ref = f3d64.filter3d(m.xyz_.double().cpu().numpy(), np.float32(_packed(dc)).astype(np.float64))
        got, want = m.filter_3D_.double().cpu().numpy(), ref["filter"]
        keep = ~ref["near"]
        err = np.abs(got - want)[keep] / (want[keep] + ref["zs"][keep] / ref["F"] * f3d64.SQRT02)
        self.worst["filter"] = max(self.worst.get("filter", 0.0), float(err.max()))
        assert err.max() < TOL_FILTER, err.max()
        self.ses.set_filter(m.filter_3D_.double().clone())

    def densify(self):
        m = self.m
        if self.dp is not None:
            self.tr.gather_moments()
            self.tr.sync_densify_stats()
        r0 = _rows(m)
        g = (r0["accum"] / r0["denom"]).nan_to_num(0.0).reshape(-1)
        max_grad = _gap(g[g > 0].cpu().numpy(), 0.85)
        extent = _gap(torch.exp(r0["p"][4]).max(1).values.cpu().numpy(), 0.5) / m.percent_dense_
        ns = m.densifySplitCount(max_grad, extent)
        z = torch.randn((2 * ns, 3), device=self.dev, generator=torch.Generator(device=self.dev).manual_seed(self.n))
        want, parents, K0 = session64.densify(r0, z.double(), max_grad, 0.0, extent, 0, m.percent_dense_, self.ses.conv)
        P0 = m.num_points()
        counts = m.densifyAndPrune(max_grad, 0.0, extent, 0, samples=z)
        torch.cuda.synchronize()
        assert counts[0] == want["p"][0].shape[0] > P0 and counts[1] == K0 and counts[4] == ns and counts[2] > 0, counts
        self.splits += ns
        new = torch.arange(K0, counts[0], device=self.dev)
        rows = torch.zeros(counts[0], dtype=torch.bool, device=self.dev)
        rows[K0 + counts[2]:] = True                          # the split children: xyz and scaling computed
        errs = self.check_rows(want, {0: (rows, 1e-6, 1e-6), 4: (rows, 1e-6, 1e-6)}, new if self.ses.conv.new_moments_zero else None)
        self.sizes.append(m.num_points())
        self.filter3d()
        return errs

    def prune(self, P_floor):
        """~30 % of the rows, leaving fewer than P_floor and a P that is 1 or 3 mod 4"""
        m = self.m
        P = m.num_points()
        n = int(0.3 * P)
        while (P - n) % 4 not in (1, 3) or P - n >= P_floor:
            n += 1
        gen = torch.Generator(device=self.dev).manual_seed(77 + self.n)
        mask = torch.zeros(P, dtype=torch.bool, device=self.dev)
        mask[torch.randperm(P, device=self.dev, generator=gen)[:n]] = True
        want = session64.prune(_rows(m), mask)
        m.prunePoints(mask)
        self.exact(self.check_rows(want))
        assert P // 128 > m.num_points() // 128 + 1 and m.num_points() < P_floor
        self.sizes.append(m.num_points())
        self.filter3d()

    def reset_opacity(self):
        m = self.m
        r0 = _rows(m)
        want = session64.reset_opacity(r0)
        m.resetOpacity()
        torch.cuda.synchronize()
        # logit(sigmoid(o)) through float32: a few roundings of sigmoid(o), amplified by logit's slope 1 / (p (1 - p))
        p = torch.sigmoid(r0["p"][3])
        self.exact(self.check_rows(want, {3: (torch.ones(m.num_points(), dtype=torch.bool, device=self.dev), 1e-6, 2.0 ** -22 / (p * (1 - p)))}))

    def transform(self):
        m = self.m
        a = 0.02
        T = np.eye(4)
        T[:3, :3] = [[math.cos(a), -math.sin(a), 0.0], [math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]]
        T[:3, 3] = [0.01, -0.02, 0.03]
        T = np.float32(T).astype(np.float64)
        want = session64.transform(_rows(m), 1.01, T)
        m.applyScaledTransformation(1.01, torch.from_numpy(np.float32(T)))
        torch.cuda.synchronize()
        allr = torch.ones(m.num_points(), dtype=torch.bool, device=self.dev)
        self.exact(self.check_rows(want, {0: (allr, 1e-5, 1e-5), 4: (allr, 1e-6, 1e-7)}))
        self.filter3d()

    def spread(self, rows):
        """New rows made by the insert recipe sit on two decisions the step cannot be measured across, and the settling jitter of xyz and
        opacity does not move them: an isotropic scale (the render does not see the rotation, so its true gradient is zero and Adam's first
        step normalises float32 noise) and a view-independent colour, exactly the target pixel's, that may lie at the clamp at 0. After the
        surgery's check, their log-scales are spread and a colour within 0.01 of the clamp is moved to 0.02, so that the next step measures
        every row."""
        m = self.m
        gen = torch.Generator(device=self.dev).manual_seed(300 + self.n)
        m.scaling_[rows] += 0.2 * torch.randn((int(rows.sum()), 3), device=self.dev, generator=gen)
        dc = m.features_dc_[rows]
        m.features_dc_[rows] = torch.where((dc * session64.SH_C0 + 0.5).abs() < 0.01, (0.02 - 0.5) / session64.SH_C0, dc)

    def insert(self):
        """increasePcd of 301 points inside the first view"""
        m = self.m
        rng = np.random.default_rng(self.n)
        fx = W / (2.0 * float(self.cams[0]["tanfovx"]))
        z = rng.uniform(1.0, 6.0, 301)
        u, v = rng.uniform(0, W, 301), rng.uniform(0, H, 301)
        pts = torch.tensor(np.stack([(u - 0.5 * (W - 1)) / fx * z, (v - 0.5 * (H - 1)) / fx * z, z], 1), dtype=torch.float32, device=self.dev)
        cols = torch.tensor(rng.uniform(0, 1, (301, 3)), dtype=torch.float32, device=self.dev)
        P = m.num_points()
        want = session64.insert_points(_rows(m), pts.double(), cols.double())
        m.increasePcd(pts, cols, iteration=self.n)
        torch.cuda.synchronize()
        rows = torch.zeros(P + 301, dtype=torch.bool, device=self.dev)
        rows[P:] = True
        # the per-operation test's tolerances (test_densify_gpu): f_dc 1e-6, the 3-NN scale 1e-6 (here against float64: 1e-5), opacity 1e-6
        self.exact(self.check_rows(want, {1: (rows, 1e-6, 1e-6), 3: (rows, 1e-6, 1e-6), 4: (rows, 1e-5, 1e-6)}, rows))
        self.spread(rows)
        self.sizes.append(m.num_points())
        self.filter3d()

    def seed(self):
        """seedFromDepth on the first view's depth target: at most 97 rows on a stride-2 grid"""
        m, tr = self.m, self.tr
        cam, c = self.cam(0), self.c(0)
        A, D = torch.empty((H, W), device=self.dev), torch.empty((H, W), device=self.dev)
        tr.render(c, out_depth=D, out_alpha=A)
        torch.cuda.synchronize()
        np_ = lambda t: t.double().cpu().numpy()
        plan = seed64.seed(cam, np_(A), np_(D), np_(self.tg["depth"]), np_(self.tg["gt"]), np_(self.tg["mask"]), stride=2, max_new=97)
        P = m.num_points()
        want = session64.seed_rows(_rows(m), plan)
        n, holes, front = tr.seedFromDepth(c, self.tg["gt"], self.tg["depth"], mask=self.tg["mask"], stride=2, max_new=97)
        torch.cuda.synchronize()
        assert n == plan["n"] > 0 and (holes, front) == plan["counts"][1:], (n, holes, front, plan["counts"])
        rows = torch.zeros(P + n, dtype=torch.bool, device=self.dev)
        rows[P:] = True
        scale = max(1.0, float(np.abs(plan["xyz"]).max()))
        # test_seed_gpu's tolerances
        self.exact(self.check_rows(want, {0: (rows, 1e-6, 1e-6 * scale), 1: (rows, 1e-6, 1e-6), 3: (rows, 1e-6, 1e-6), 4: (rows, 1e-5, 1e-6)}, rows))
        self.spread(rows)
        self.sizes.append(m.num_points())
        self.filter3d()

    def relocate_grow(self):
        """the pair mcmcRefine runs, with injected uniforms: 40 rows made dead are relocated, then the map grows by 5 %"""
        m = self.m
        m._exist()
        gen = torch.Generator(device=self.dev).manual_seed(5)
        m.opacity_[torch.randperm(m.num_points(), device=self.dev, generator=gen)[:40]] = -8.0
        before = _host(m)
        w = _w32(before["p"][3][:, 0])
        dead = int((w <= MIN_OP).sum())
        u = _safe_uniforms(np.where(w > MIN_OP, w, 0.0), dead, 3)
        want, picks, dead_rows = session64.relocate(before, u, MIN_OP, self.n, self.ses.conv)
        assert m.relocateGaussians(MIN_OP, iteration=self.n, uniforms=torch.from_numpy(u)) == dead == len(dead_rows) >= 40
        torch.cuda.synchronize()
        _compare_mcmc(m, before, want, picks, dead_rows, self.n, m.num_points())     # test_mcmc_gpu's checks and tolerances
        before = _host(m)
        P = m.num_points()
        P_new = int(math.floor(1.05 * P))
        u = _safe_uniforms(_w32(before["p"][3][:, 0]), P_new - P, 4)
        want, picks = session64.grow(before, P_new, u, MIN_OP, self.n, self.ses.conv)
        assert m.addNewGaussians(10 ** 6, 1.05, MIN_OP, iteration=self.n, uniforms=torch.from_numpy(u)) == P_new - P
        torch.cuda.synchronize()
        _compare_mcmc(m, before, want, picks, np.arange(P, P_new), self.n, P)
        self.sizes.append(m.num_points())
        self.filter3d()

    def setters(self):
        """every set*LearningRate on the model and in the truth; the xyz one holds until the next updateLearningRate"""
        m, s = self.m, self.ses
        for name, group, lr in (("Feature", "features_dc", 0.002), ("Opacity", "opacity", 0.03), ("Scaling", "scaling", 0.004),
                                ("Rotation", "rotation", 0.0015), ("Position", "xyz", 1.1e-4)):
            getattr(m, f"set{name}LearningRate")(lr)
            s.set_lr(group, lr)

    def set_sh(self, D):
        self.m.setShDegree(D)
        self.ses.set_sh(D)

    def edges(self):
        """the session passed through a shrink below a size seen before followed by a grow, a crossing of a multiple of 128, and a
        step at D = 3"""
        s = self.sizes
        shrink_then_grow = any(s[j] < min(s[:j]) and max(s[j + 1:], default=0) > s[j] for j in range(1, len(s)))
        crossed = any(a // 128 != b // 128 for a, b in zip(s, s[1:]))
        assert shrink_then_grow and crossed and self.d3, (s, self.d3)


# ---- GaussianTrainer sessions -------------------------------------------------------------------------------------------------------
# (flag set k as in test_step64_gpu: depth = bit 0, aa = 1, reg = 2, f3d = 3, normal = 4; deterministic; scene)
SESSIONS = [(0, False, "terminate"), (1, True, "clamp"), (6, False, "terminate"), (8, True, "clamp"), (17, False, "terminate"),
            (14, True, "clamp"), (31, False, "terminate"), (19, True, "clamp")]


@pytest.mark.parametrize("k,det,scene", SESSIONS, ids=[f"{k}-{step64.flag_name(step64.ALL_FLAGS[k])}-{'det' if d else 'fast'}" for k, d, _ in SESSIONS])
def test_session(cuda, k, det, scene):
    fl = step64.ALL_FLAGS[k]
    r = Run(cuda, fl, det, scene)
    r.step()
    r.step()
    P0 = r.m.num_points()
    r.exact(r.densify())
    r.step()
    r.dn_step()
    r.step()
    r.prune(P0)
    r.step()
    r.dist_step()
    r.step()
    r.insert()
    r.step()
    r.setters()
    r.set_sh(3)
    r.step(schedule=False)
    r.render()
    r.step()
    r.reset_opacity()
    r.step()
    r.transform()
    r.step()
    r.backward_pixels()
    r.step()
    r.seed()
    r.step()
    if fl.reg:
        r.relocate_grow()
        r.step()
    r.edges()
    assert r.splits > 0, "the session must split rows"
    print(f"MEASURED session {k} {step64.flag_name(fl)} det={det} sizes={r.sizes} excluded={r.excl} {r.worst}")
    _assert_gates({q: v for q, v in r.worst.items() if q != "filter"}, GATE_STEP_TRAJ)


def test_sessions_cover_the_flags_modes_and_rows():
    fls = [step64.ALL_FLAGS[k] for k, _, _ in SESSIONS]
    for name in ("depth", "aa", "reg", "f3d", "normal"):
        assert {getattr(f, name) for f in fls} == {False, True}, name
    assert {d for _, d, _ in SESSIONS} == {False, True}


# ---- DataParallelTrainer sessions at world 1 ----------------------------------------------------------------------------------------
DP_SESSIONS = [(p, d) for p in ("p2p", "nccl", "slabs") for d in (False, True)]
DP_KW = {"p2p": dict(mode="p2p"), "nccl": dict(mode="nccl", pipeline=False), "slabs": dict(mode="nccl", pipeline=True, nslabs=3)}
DP_KW = {k: dict(v, deterministic=True) for k, v in DP_KW.items()}     # the same gradients on every run of the file


def _frozen(m):
    return [t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + [m.xyz_gradient_accum_, m.denom_, m.max_radii2D_]] + [m.step_]


@pytest.mark.parametrize("path,depth", DP_SESSIONS, ids=[f"{p}-{'depth' if d else 'nodepth'}" for p, d in DP_SESSIONS])
def test_dp_session(cuda, path, depth):
    fl = step64.Flags(depth=depth)
    r = Run(cuda, fl, False, "terminate" if depth else "clamp", dp=DP_KW[path])
    assert r.tr.mode == DP_KW[path]["mode"] and (path == "p2p" or r.tr.pipeline == (path == "slabs"))
    r.step()
    r.step()
    P0 = r.m.num_points()
    r.exact(r.densify())
    # a step over the resized model without rebuild() is refused before it touches anything
    before, it = _frozen(r.m), r.tr.iteration
    with pytest.raises(ValueError, match="rebuild"):
        r.tr.trainForOneIteration(r.c(), r.tg["gt"], r.tg["mask"])
    torch.cuda.synchronize()
    after = _frozen(r.m)
    assert all(torch.equal(a, b) for a, b in zip(before[:-1], after[:-1])) and before[-1] == after[-1] and r.tr.iteration == it
    r.tr.rebuild()
    r.tr.render(r.c())
    r.step()
    r.step()
    r.tr.gather_moments()
    r.prune(P0)
    r.tr.rebuild()
    r.tr.render(r.c())
    r.step()
    r.exact(r.densify())               # gather_moments and sync_densify_stats first; P grows back into the freed capacity
    r.tr.rebuild()
    r.tr.render(r.c())
    r.set_sh(3)
    r.step()
    r.edges()
    if path == "p2p":
        r.tr.close()
    print(f"MEASURED dp session {path} {step64.flag_name(fl)} sizes={r.sizes} excluded={r.excl} {r.worst}")
    _assert_gates(r.worst, GATE_STEP_TRAJ)


# ---- the gates bite -----------------------------------------------------------------------------------------------------------------
def test_perturbed_new_rows_inherit_moments(cuda):
    r = Run(cuda, step64.ALL_FLAGS[0], False, "terminate", conv=session64.SessionConv(new_moments_zero=False))
    r.step()
    errs = r.densify()
    err = max(v for q, v in errs.items() if q.startswith("mom"))
    print(f"MEASURED perturbed inherit: {err:.2e} (gate {GATE_MOM:.0e})")
    assert err > GATE_MOM


def test_perturbed_xyz_lr_held(cuda):
    r = Run(cuda, step64.ALL_FLAGS[0], False, "terminate", conv=session64.SessionConv(lr_schedule=False))
    r.m.step_ = 8                      # lr(8) = 0.54 lr_init
    st, res = _perturbed_step(r)
    err = _step_err(r.m.xyz_, res["state"]["params"]["xyz"], st["lr"][0])
    print(f"MEASURED perturbed lr-held: {err:.2e} (gate {GATE_STEP_TRAJ:.0e})")
    assert err > GATE_STEP_TRAJ


def _perturbed_step(r):
    """one step of the kernels and of the (perturbed) truth -> (the truth's state before it, its result)"""
    m, fl = r.m, r.fl
    m.updateLearningRate(m.step_)
    r.ses.update_lr(m.step_)
    st, cam64, _ = _settled_state(m, fl, r.cam(), r.tg64, 5, 0)
    r.loss = _kernel_step(r.tr, m, r.c(), r.tg, fl, 0)
    return r.ses.state(st), r.ses.step(st, cam64, r.tg64, fl)


def _loss_err(r):
    """-> the largest relative error of the loss scalars of one step against the (perturbed) truth"""
    _, res = _perturbed_step(r)
    return max(abs(a - res["loss"][q]) / abs(res["loss"][q]) for a, q in zip(r.loss, ("loss", "l1", "ssim")))


def test_perturbed_stale_filter(cuda):
    r = Run(cuda, step64.ALL_FLAGS[8], True, "clamp", conv=session64.SessionConv(filter_current=False))
    r.step()
    r.transform()
    err = _loss_err(r)
    print(f"MEASURED perturbed stale-filter: {err:.2e} (gate {GATE_LOSS:.0e})")
    assert err > GATE_LOSS


def test_perturbed_sh_degree_left_at_2(cuda):
    r = Run(cuda, step64.ALL_FLAGS[0], False, "terminate", conv=session64.SessionConv(sh_raise=False))
    r.set_sh(3)
    err = _loss_err(r)
    print(f"MEASURED perturbed sh-at-2: {err:.2e} (gate {GATE_LOSS:.0e})")
    assert err > GATE_LOSS
