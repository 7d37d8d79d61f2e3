"""Shared helpers for the parity tests: scene -> device tensors, and the stored outputs of the reference build
(tests/golden/<module>.npz, written by tests/golden/make_ref_golden.py) that the GPU parity tests compare against."""
import hashlib
import os

import numpy as np
import torch

import photo_slam_b200.synthetic as syn


def scene_tensors(P, camname="tum", seed=0, pose_seed=None, dev="cuda", scale=1.0, wh=None, scale_px=2.4):
    W, H, fx, fy = syn.CAMERAS[camname]
    if wh is not None:
        fx, fy = fx * wh[0] / W, fy * wh[1] / H
        W, H = wh
    R = t = None
    if pose_seed is not None:
        R, t = syn.random_pose(np.random.default_rng(pose_seed))
    cam = syn.make_camera(W, H, fx, fy, R, t)
    sc = syn.make_scene(P, cam, seed=seed, scale_px=scale_px)
    act = syn.activate(sc)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    g = {k: T(v) for k, v in act.items()}
    c = syn.device_camera(cam, dev)
    return cam, sc, act, g, c


def rel_close(a, b, rtol=1e-4, atol=1e-7):
    """SURVEY §8(d) float gate: |a-b| <= rtol*max(|a|,|b|) + atol. Returns fraction of elements violating it."""
    a = a.double().flatten()
    b = b.double().flatten()
    bad = (a - b).abs() > (rtol * torch.maximum(a.abs(), b.abs()) + atol)
    return bad.double().mean().item() if a.numel() else 0.0


# tests/golden/ref_small.npz: the reference's outputs and intermediates for these seeded scenes (tests/golden/make_golden.py)
ORACLE_CASES = {"a": dict(P=1500, wh=(128, 80), pose_seed=3, D=3, bg=(0.1, 0.2, 0.3), scale_px=4.0, seed=7),
                "b": dict(P=600, wh=(75, 41), pose_seed=8, D=1, bg=(0.0, 0.0, 0.0), scale_px=7.0, seed=9)}

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SAMPLE = 2048   # elements kept per stored array; integer and bit-exact gates compare a SHA-1 of the whole array instead


def sample_index(n, k=SAMPLE):
    """Fixed, seeded element positions of a flattened array of n elements (all of them when n <= k)."""
    if n <= k:
        return np.arange(n)
    return np.sort(np.random.default_rng(n).choice(n, k, replace=False))


def _np(t):
    return np.ascontiguousarray(t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t))


def digest(t):
    a = _np(t)
    return hashlib.sha1(a.tobytes()).hexdigest()


def compact(case, out, digest_only=()):
    """{name: tensor | scalar} of one reference run -> npz entries: whole-array digest, size and a seeded sample per tensor
    (no sample for the names in digest_only, which are only ever compared bit for bit)."""
    d = {f"{case}/#present": np.array(1)}
    for k, v in out.items():
        if torch.is_tensor(v) or (isinstance(v, np.ndarray) and v.ndim > 0):
            a = _np(v).reshape(-1)
            d[f"{case}/{k}#sha"] = np.array(digest(v))
            d[f"{case}/{k}#n"] = np.array(a.size)
            if k not in digest_only:
                d[f"{case}/{k}#s"] = a[sample_index(a.size)]
        else:
            d[f"{case}/{k}"] = np.array(v)
    return d


class Gold:
    """The reference's outputs for one case of a parity test, as stored by compact()."""

    def __init__(self, module, case):
        path = os.path.join(GOLDEN_DIR, module + ".npz")
        z = np.load(path)
        self.case, self.z = case, z
        if f"{case}/#present" not in z.files:
            raise KeyError(f"{path} has no case {case!r}: regenerate it with tests/golden/make_ref_golden.py")

    def __getitem__(self, name):
        v = self.z[f"{self.case}/{name}"]
        return v.item() if v.ndim == 0 else v

    def exact(self, name, t):
        """t has the stored size and the same bits as the reference's array."""
        return int(t.numel()) == int(self.z[f"{self.case}/{name}#n"]) and digest(t) == str(self.z[f"{self.case}/{name}#sha"])

    def pair(self, name, t):
        """(mine, reference) at the stored sample positions, as float64 tensors on t's device."""
        assert int(t.numel()) == int(self.z[f"{self.case}/{name}#n"]), f"{name}: {t.numel()} elements, reference has {self.z[f'{self.case}/{name}#n']}"
        idx = torch.from_numpy(sample_index(t.numel())).to(t.device)
        ref = torch.from_numpy(self.z[f"{self.case}/{name}#s"].astype(np.float64)).to(t.device)
        return t.reshape(-1)[idx].double(), ref

    def full(self, name):
        """A stored array small enough to have been kept whole."""
        n, a = int(self.z[f"{self.case}/{name}#n"]), self.z[f"{self.case}/{name}#s"]
        assert a.size == n, f"{name}: only a sample of {n} elements is stored"
        return a

    def frac(self, name, t, rtol=1e-4, atol=1e-7):
        """rel_close over the stored sample."""
        return rel_close(*self.pair(name, t), rtol=rtol, atol=atol)

    def relnorm(self, name, t):
        """|mine - reference| / |reference| over the stored sample."""
        a, b = self.pair(name, t)
        return ((a - b).norm() / (b.norm() + 1e-30)).item()
