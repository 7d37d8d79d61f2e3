"""-m gpu: the kernels against the float64 truth at the sizes bench.py runs, on a seeded sample of tiles (tests/scale64.py).

Scenes are bench.py's own (syn.make_scene(P, cam, seed=0) in front of the identity view) plus three built to reach what they do not:
  * B: 500k at 1200x680 (75 x 43 tiles, 12 tile-id bits, two tile-sort passes), and its 600x340 and 300x170 pyramid levels, whose last
    tile row and column are partial; C: 1M at 640x480; D: 3M at 1200x680 (about 2900 emit blocks, lists of about 4000 entries);
  * deep: B plus an 11000-splat cluster over one tile: a list of more than 8192 entries, pixels whose T crosses 1e-4 past list position
    2000, and 0.99 clamps past position 1000;
  * sky: B plus 300 splats each over more than 100 tiles (non-tight lists, beyond TIGHT_MAX_AREA), half of them at low opacity, at
    neighbouring depths, so that 1024 depth-consecutive Gaussians hold more than EM_STAGE instances;
  * wide: 300k sparse at 4100x4100: 257 x 257 tiles with partial edges, 17 tile-id bits and three tile-sort passes.
Each scene asserts that it reaches its path, from psb_debug_export (list lengths, contributor counts) and the truth's geometry.

Cases: the operator (RasterizeGaussiansDepthCUDA, plain and anti-aliased; atomic and deterministic backward); the trainer's render and
backwardPixels(grads=...) in each of the 24 tile-backward variants it dispatches (anti-aliasing on and off, the 3D filter once); Adam mode
(backwardPixels(grads=None)) from seeded moments, once after an overflow of the initial binning arena; a second deterministic pass over
another view; and perturbed truths that the operator's and the trainer's gates must reject.

Gates: per pixel, |kernel - truth| <= a + b n, n = the pixel's contributor count, measured on an H100 SXM (80 GB, 700 W); the largest
measured value sits beside each gate. Gradients are gated on the candidate rows by rel-norm and by the largest element error relative
to the group's largest element, and every other row must be exactly zero.
"""
import numpy as np
import pytest
import torch

import photo_slam_b200.synthetic as syn
import scale64
import splat64 as s64
import step64
from test_splat64_gpu import _debug_state, _export, _maxerr, _model, _op_forward, _relnorm

pytestmark = pytest.mark.gpu

# Per-pixel forward gate a L + b n: L = max(W, H), n = the pixel's contributor count; colour, normal, A and final T absolute, depth and
# depth2 relative to the largest truth value of the sample. Both terms are measured (normal plane, the largest): 5.6e-5 at L = 4100
# with n < 100 (wide) and 1.6e-5 at L = 1200 with n < 100 (B), i.e. 1.4e-8 L from the float32 pixel coordinate; 1.4e-5 at L = 300
# with n < 2000 (B-300x170), i.e. 7e-9 n from the blend. At n >= 2000 (deep) at most 8.9e-6: no faster than linear in n.
GATE_PIX_A, GATE_PIX_B = 2.5e-8, 1e-8
GATE_GRAD = 1e-4          # rel-norm per group on the candidate rows: measured 4.8e-5 (operator wide, scales); 1.3e-5 at 1200 px
GATE_GRAD_MAX = 2e-4      # max |kernel - truth| / max |truth| per group: measured 8.7e-5 (operator wide, scales); 1.9e-5 at 1200 px
N_TILES = 48
EM_STAGE = 5120                           # psb_forward.cu: instances staged per emit block
TIGHT_MAX_AREA = 32                       # psb_common.cuh


# ---- scenes -------------------------------------------------------------------------------------------------------------------------
def _bench(P, cam_name, W=None, H=None):
    Wc, Hc, fx, fy = syn.CAMERAS[cam_name]
    cam0 = syn.make_camera(Wc, Hc, fx, fy)
    sc = syn.make_scene(P, cam0, seed=0)
    if W is None:
        return cam0, sc
    s = W / Wc
    return syn.make_camera(W, H, fx * s, fy * s), sc


def _off_near(sc):
    """identity view: move Gaussians within 1e-3 (relative) of the near plane off it (tile_truth refuses a splat on it)"""
    z = sc["xyz"][:, 2]
    on = np.abs(z - s64.NEAR) < 1e-3 * s64.NEAR
    sc["xyz"][on, 2] = np.where(z[on] > s64.NEAR, 0.21, 0.19).astype(np.float32)


def _put(sc, cam, idx, u, v, z, sigma_px, logit):
    fx = cam["W"] / (2.0 * float(cam["tanfovx"]))
    sc["xyz"][idx] = np.stack([(u - 0.5 * cam["W"]) / fx * z, (v - 0.5 * cam["H"]) / fx * z, z], 1)
    sc["scaling"][idx] = np.log(sigma_px / fx * z)[:, None]
    sc["rotation"][idx] = [1.0, 0.0, 0.0, 0.0]
    sc["opacity"][idx] = np.asarray(logit, np.float32).reshape(-1, 1)


def _append(sc, n):
    P = sc["xyz"].shape[0]
    for k, v in sc.items():
        sc[k] = np.ascontiguousarray(np.concatenate([v, np.repeat(v[:1], n, 0)], 0))
    return np.arange(P, P + n)


def _deep():
    cam, sc = _bench(500_000, "replica")
    rng = np.random.default_rng(11)
    n = 11000                # enough instances that a fresh trainer's first pass overflows its initial arena (6 P + 65536)
    idx = _append(sc, n)
    u0, v0 = 37 * 16 + 8.0, 21 * 16 + 8.0
    # in front of every bench Gaussian (z >= 0.5), wide and faint: alpha 0.0041-0.0045 on the whole tile, so T reaches 1e-4 after
    # about 2100 blends
    z = 0.3 + 0.2 * (np.arange(n) + rng.uniform(0.2, 0.8, n)) / n
    _put(sc, cam, idx, u0 + rng.uniform(-2, 2, n), v0 + rng.uniform(-2, 2, n), z, rng.uniform(30.0, 40.0, n), np.full(n, -5.4))
    sc["scaling"][idx] += np.log(rng.uniform(0.85, 1.0, (n, 3))).astype(np.float32)     # anisotropic: disc far above its 0.1 clamp
    sc["rotation"][idx] = rng.normal(size=(n, 4)).astype(np.float32)
    # a few opaque narrow splats deep in the list, on pixel centres offset by 0.05: alpha reaches the 0.99 clamp there
    k = idx[1200:1210]
    _put(sc, cam, k, u0 - 7 + 1.5 * np.arange(10) + 0.05, np.full(10, v0 + 0.05), z[1200:1210], np.full(10, 1.5), np.full(10, 6.0))
    return dict(cam=cam, sc=sc, must=[(37, 21)], edge="deep")


def _sky():
    cam, sc = _bench(500_000, "replica")
    rng = np.random.default_rng(12)
    n = 300
    idx = _append(sc, n)
    u, v = rng.uniform(100, 1100, n), rng.uniform(80, 600, n)
    logit = np.where(np.arange(n) % 2 == 0, -3.0, rng.uniform(-1.0, 1.0, n))
    _put(sc, cam, idx, u, v, 3.0 + 2e-4 * np.arange(n) + 2e-5 * rng.uniform(size=n), rng.uniform(40.0, 80.0, n), logit)
    must = [(int(u[i]) // 16, int(v[i]) // 16) for i in range(0, n, 60)]
    return dict(cam=cam, sc=sc, must=must, edge="sky")


def _wide():
    W = H = 4100
    cam = syn.make_camera(W, H, 3000.0, 3000.0)
    sc = syn.make_scene(300_000, cam, seed=0)
    return dict(cam=cam, sc=sc, must=[], edge="wide")


SCENES = {"B": lambda: dict(zip(("cam", "sc"), _bench(500_000, "replica")), must=[], edge=None),
          "B-600x340": lambda: dict(zip(("cam", "sc"), _bench(500_000, "replica", 600, 340)), must=[], edge=None),
          "B-300x170": lambda: dict(zip(("cam", "sc"), _bench(500_000, "replica", 300, 170)), must=[], edge=None),
          "C": lambda: dict(zip(("cam", "sc"), _bench(1_000_000, "tum")), must=[], edge=None),
          "D": lambda: dict(zip(("cam", "sc"), _bench(3_000_000, "replica")), must=[], edge=None),
          "deep": _deep, "sky": _sky, "wide": _wide}
_CACHE = {}


def _scene(name):
    if name not in _CACHE:
        s = SCENES[name]()
        _off_near(s["sc"])
        _CACHE[name] = s
    return _CACHE[name]


def _tiles(s, list_len, nc):
    """the sample: the scene's own tiles, the longest list, the deepest last contributor, partial edge tiles, then seeded ones"""
    W, H = s["cam"]["W"], s["cam"]["H"]
    gx = -(-W // 16)
    longest = int(torch.argmax(list_len))
    deepest = int(torch.argmax(nc.reshape(-1)))
    must = list(s["must"]) + [(longest % gx, longest // gx), ((deepest % W) // 16, (deepest // W) // 16)]
    return scale64.sample_tiles(W, H, N_TILES, seed=0, must=must)


def _check_reach(name, s, tiles, t, list_len, nc):
    W, H = s["cam"]["W"], s["cam"]["H"]
    ntiles = (-(-W // 16)) * (-(-H // 16))
    bits = int(np.ceil(np.log2(ntiles)))
    assert bits > 8 or name.startswith("B-"), name      # the pyramid levels are there for their partial tiles
    gx = -(-W // 16)
    ll = list_len[[ty * gx + tx for tx, ty in tiles]]
    if s["edge"] == "wide":
        assert bits > 16
    if s["edge"] == "deep":
        assert int(ll.max()) > 8192 and int(nc.max()) > 2000
        deep = t["n_contrib"] > 2000
        assert (deep & t["stopped"]).any(), "a pixel whose T crosses 1e-4 past position 2000"
        assert (t["clamped"] & (t["n_contrib"] > 1000)).any(), "a 0.99 clamp past position 1000"
    if s["edge"] == "sky":
        assert int(t["tiles_touched"][t["cand"]].max()) > 100
    print(f"MEASURED reach {name}: tile bits {bits}, longest sampled list {int(ll.max())}, deepest contributor {int(nc.max())}")


def _bound(name, t, L):
    """excluded pixels within 8 % of the sampled ones, Gaussian-level offenders within 0.1 % of P at L = max(W, H) <= 1200 (a rectangle
    edge is ambiguous within a few ulps of the pixel coordinate, which grows with L). The pixel share grows with the number of alpha
    tests per pixel: measured 1.0 % on B, 3.5 % on C (1M at 640x480), 6.9 % on D (3M at 1200x680, lists of about 4000 entries, of which
    3 % of the pixels hold an alpha test within 1e-4 of 1/255); offenders 0.05 % of P at most (0.12 % for wide at L = 4100)."""
    c = t["counts"]
    print(f"MEASURED exclusions {name}: {c}")
    return c["excluded"] <= 0.08 * c["pixels"] and c["offenders"] <= 1e-3 * c["P"] * max(1.0, L / 1200)


def _pix_gate(L, n):
    return GATE_PIX_A * L + GATE_PIX_B * n.double()


def _pixel_errs(name, what, err, n, L):
    """per-pixel error against a L + b n; prints the largest error in bins of n"""
    gate = _pix_gate(L, n)
    bins = {}
    for lo, hi in ((0, 100), (100, 500), (500, 2000), (2000, 10 ** 9)):
        m = (n >= lo) & (n < hi)
        if m.any():
            bins[f"n<{hi}" if hi < 10 ** 9 else "n>=2000"] = f"{float(err[m].max()):.2e}"
    print(f"MEASURED {name} {what} per-pixel max by n: {bins}, worst ratio to gate {float((err / gate).max()):.3f}")
    return bool((err <= gate).all())


def _grad_errs(errs, key, a, ref, cand):
    a, ref = a.double(), ref.double()
    other = torch.ones(a.shape[0], dtype=torch.bool, device=a.device)
    other[cand] = False
    assert not a[other].any(), f"{key}: a gradient on a row no sampled tile reaches"
    if not ref[cand].any():         # a group the truth leaves at zero must be zero, not skipped
        assert not a.any(), f"{key}: a gradient where the truth has none"
        return
    errs[f"grad-{key}"] = _relnorm(a[cand], ref[cand])
    errs[f"gradmax-{key}"] = _maxerr(a[cand], ref[cand], float(ref[cand].abs().max()))


def _weights(H, W, dev, keep, seed=0):
    gen = torch.Generator().manual_seed(seed)
    r = lambda *sh: (torch.rand(sh, generator=gen) - 0.5).to(dev)
    w = dict(color=r(3, H, W), depth=0.2 * r(H, W), alpha=r(H, W), normal=r(3, H, W), depth2=0.02 * r(H, W))
    return {k: (v * keep).float().contiguous() for k, v in w.items()}


# ---- the operator -------------------------------------------------------------------------------------------------------------------
def _op_inputs(sc, dev):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in syn.activate(sc).items()}


OP_CASES = [("B", False), ("B", True), ("B-600x340", False), ("B-300x170", True), ("C", True), ("D", False), ("deep", False), ("sky", True),
            ("wide", False)]


def _op_pass(cuda, name, aa, perturb=None):
    from photo_slam_b200 import rasterizer
    s = _scene(name)
    cam = s["cam"]
    c, g = syn.device_camera(cam, cuda), _op_inputs(s["sc"], cuda)
    bg = (0.0, 0.0, 0.0)
    bgt = torch.zeros(3, device=cuda)
    P, W, H = g["means3D"].shape[0], cam["W"], cam["H"]
    R, color, depth, radii, geom, binning, img = _op_forward(g, c, bgt, 3, aa)
    tt, list_len, nc = _export(P, R, W, H, geom, binning, img)
    tiles = _tiles(s, list_len, nc)
    leaves = {k: v.double().requires_grad_(True) for k, v in g.items()}
    c64 = s64.camera64(cam, cuda)
    # exclusions first (no grad), then the weights masked by them for both sides
    t = scale64.tile_truth({k: v.detach() for k, v in leaves.items()}, c64, bg, tiles, D=3, aa=aa, raw=False, perturb=perturb)
    w = _weights(H, W, cuda, t["keep"])
    w = dict(color=w["color"], depth=w["depth"])
    t = scale64.tile_truth(leaves, c64, bg, tiles, D=3, aa=aa, raw=False, weights=w, perturb=perturb)
    return s, tiles, t, leaves, dict(R=R, color=color, depth=depth, radii=radii, geom=geom, binning=binning, img=img, tt=tt, list_len=list_len,
                                     nc=nc, g=g, c=c, bgt=bgt, w=w)


def _op_errs(name, s, tiles, t, k):
    W = s["cam"]["W"]
    gx = -(-W // 16)
    ok = ~t["offender"]
    disc = dict(radii=bool(torch.equal(k["radii"].long()[ok], t["radii"][ok])), tiles_touched=bool(torch.equal(k["tt"][ok], t["tiles_touched"][ok])),
                list_len=bool(torch.equal(k["list_len"][[ty * gx + tx for tx, ty in tiles]][~t["list_ambiguous"]], t["list_len"][~t["list_ambiguous"]])))
    keep = ~t["excluded"]
    n = t["n_contrib"][keep]
    sure = keep & ~t["list_ambiguous"][t["tile"]]
    disc["n_contrib"] = bool(torch.equal(k["nc"].reshape(-1)[t["pix"]][sure], t["n_contrib"][sure]))
    col = (k["color"].reshape(3, -1)[:, t["pix"]][:, keep].double() - t["color"][:, keep]).abs().amax(0)
    zmax = float(t["depth"].abs().max())
    dep = (k["depth"].reshape(-1)[t["pix"]][keep].double() - t["depth"][keep]).abs() / zmax
    return disc, dict(color=(col, n), depth=(dep, n))


@pytest.mark.parametrize("name,aa", OP_CASES, ids=[f"{n}-{'aa' if a else 'plain'}" for n, a in OP_CASES])
def test_operator_at_scale(cuda, name, aa):
    from photo_slam_b200 import rasterizer
    s, tiles, t, leaves, k = _op_pass(cuda, name, aa)
    _check_reach(name, s, tiles, t, k["list_len"], k["nc"])
    bounded = _bound(name, t, max(s["cam"]["W"], s["cam"]["H"]))
    disc, pix = _op_errs(name, s, tiles, t, k)
    assert all(disc.values()), disc
    L = max(s["cam"]["W"], s["cam"]["H"])
    ok = all(_pixel_errs(f"operator {name} aa={aa}", w, e, n, L) for w, (e, n) in pix.items())
    g, c = k["g"], k["c"]
    errs = {}
    for det in (False, True):
        out = rasterizer.RasterizeGaussiansBackwardDepthCUDA(k["bgt"], g["means3D"], k["radii"], None, g["scales"], g["rotations"], 1.0, None,
                                                             c["viewmatrix"], c["projmatrix"], c["tanfovx"], c["tanfovy"], k["w"]["color"],
                                                             k["w"]["depth"], g["shs"], 3, c["campos"], k["geom"], k["R"], k["binning"], k["img"],
                                                             deterministic=det, antialiasing=aa)
        _, _, d_op, d_m3, _, d_sh, d_sc, d_rot = out
        for key, a, ref in (("means3D", d_m3, leaves["means3D"].grad), ("shs", d_sh, leaves["shs"].grad), ("opacities", d_op, leaves["opacities"].grad),
                            ("scales", d_sc, leaves["scales"].grad), ("rotations", d_rot, leaves["rotations"].grad)):
            _grad_errs(errs, f"{key}-{'det' if det else 'atomic'}", a, ref, t["cand"])
    torch.cuda.synchronize()
    print(f"MEASURED operator {name} aa={aa} {errs}")
    assert bounded, "exclusions over their bound"
    assert ok, "a per-pixel value over its gate"
    _assert_grads(errs)


def _assert_grads(errs):
    for key, v in errs.items():
        if key.startswith("grad-"):
            assert v < GATE_GRAD, (key, v)
        if key.startswith("gradmax-"):
            assert v < GATE_GRAD_MAX, (key, v)


def _truth_list_len(geo):
    """the truth's rectangle list length of every tile (a 2D difference array over the rectangles of the live Gaussians)"""
    gx, gy = geo["gx"], geo["gy"]
    r = geo["rect"][geo["alive"]]
    cnt = torch.zeros((gy + 1, gx + 1), dtype=torch.float64, device=r.device)
    for yc, xc, sgn in ((1, 0, 1.0), (1, 2, -1.0), (3, 0, -1.0), (3, 2, 1.0)):
        cnt.index_put_((r[:, yc], r[:, xc]), torch.full((r.shape[0],), sgn, dtype=torch.float64, device=r.device), accumulate=True)
    return cnt.cumsum(0).cumsum(1)[:gy, :gx].reshape(-1)


# ---- the trainer --------------------------------------------------------------------------------------------------------------------
# The tile backward's variants (psb_render.cu launch_render_backward): base and _normal dispatch on dL_ddepth x deterministic x dL_dalpha,
# _moment on deterministic x dL_dalpha x dL_dnormal. Every one of the 24 runs once, on scenes and anti-aliasing taken in turn.
def _variants():
    out = []
    for fam in ("plain", "normal", "moment"):
        for k in range(8):
            a, b, c = bool(k & 1), bool(k & 2), bool(k & 4)
            if fam == "moment":       # (det, alpha, normal); depth weighted on odd cases of the two others
                det, alpha, normal, depth = a, b, c, bool(k % 3 == 0)
            else:
                depth, det, alpha, normal = a, b, c, fam == "normal"
            out.append((fam, depth, alpha, normal, det))
    names = ["B", "C", "deep", "sky", "wide", "B-300x170", "B-600x340", "D"]
    cases = []
    for i, (fam, depth, alpha, normal, det) in enumerate(out):
        bwd = "c" + ("d" if depth else "") + ("a" if alpha else "") + ("n" if normal else "") + ("m" if fam == "moment" else "")
        cases.append((names[i % len(names)], fam, bwd, bool(i % 2), det, i == 11))
    return cases


TR_CASES = _variants()


def _trainer(s, cuda, aa, det, f3d, c):
    from photo_slam_b200 import trainer
    m = _model(s["sc"], cuda, 3)
    f = None
    if f3d:
        m.computeFilter3D([c])
        f = m.filter_3D_.double().reshape(-1)
    tr = trainer.GaussianTrainer(m, background=torch.zeros(3, device=cuda), deterministic=det, antialiasing=aa, filter3d=f3d)
    return m, tr, f


def _num_rendered(tr, W, H, dev):
    import ctypes as C
    from photo_slam_b200 import _lib
    n = C.c_int(0)
    _lib.check(tr.L.psb_trainer_debug_state(tr.h, W, H, None, None, C.byref(n), torch.cuda.current_stream().cuda_stream), "psb_trainer_debug_state")
    return int(n.value)


def _render(tr, c, fam, bwd, dev):
    """render with the planes the backward variant needs -> kernel outputs, last and final T of psb_trainer_debug_state"""
    W, H = c["W"], c["H"]
    P = tr.model.num_points()
    k = dict(img=torch.empty((3, H, W), device=dev), rad=torch.zeros(P, dtype=torch.int32, device=dev), dep=torch.empty((H, W), device=dev),
             A=torch.empty((H, W), device=dev), N=torch.empty((3, H, W), device=dev) if "n" in bwd or fam == "normal" else None,
             M=torch.empty((H, W), device=dev) if fam == "moment" else None)
    tr.render(c, k["img"], k["rad"], out_depth=k["dep"], out_alpha=k["A"], out_normal=k["N"], out_depth2=k["M"])
    k["last"], k["fT"] = _debug_state(tr, W, H, dev)
    k["R"] = _num_rendered(tr, W, H, dev)
    return k


def _trainer_tiles(s, cam, c, aa, raw, f, cuda):
    """the sample: the scene's tiles, the longest of the truth's rectangle lists and the deepest last contributor of the operator's
    rectangle lists on the same view (the trainer's own lists are tight, so neither is readable from it)"""
    c64 = s64.camera64(cam, cuda)
    with torch.no_grad():
        geo = s64.geometry(scale64._inputs({k: v.detach() for k, v in raw.items()}, True, f), c64, 3, aa)
    ll = _truth_list_len(geo)
    longest = int(ll.argmax())
    g = _op_inputs(s["sc"], cuda)
    P, W, H = g["means3D"].shape[0], cam["W"], cam["H"]
    R, _, _, _, geom, binning, img = _op_forward(g, c, torch.zeros(3, device=cuda), 3, aa)
    _, _, nc = _export(P, R, W, H, geom, binning, img)
    deepest = int(nc.reshape(-1).argmax())
    must = s["must"] + [(longest % geo["gx"], longest // geo["gx"]), ((deepest % W) // 16, (deepest // W) // 16)]
    return scale64.sample_tiles(W, H, N_TILES, 0, must)


def _planes(fam, bwd):
    return ("color", "depth", "alpha") + (("normal",) if fam == "normal" or "n" in bwd else ()) + (("depth2",) if fam == "moment" else ())


def _weighted(w, bwd):
    keys = dict(c="color", d="depth", a="alpha", n="normal", m="depth2")
    return {keys[ch]: w[keys[ch]] for ch in bwd}


def _truths(s, cam, cuda, tiles, aa, f, planes, bwd, seed=1, perturb=None, with_grad=True):
    """(kept-pixel weights the kernel sees, the truth with its gradients on float64 raw leaves, the leaves)"""
    raw = {k: v.requires_grad_(True) for k, v in s64.raw64(s["sc"], cuda).items()}
    c64 = s64.camera64(cam, cuda)
    t0 = scale64.tile_truth({k: v.detach() for k, v in raw.items()}, c64, (0.0, 0.0, 0.0), tiles, D=3, aa=aa, f=f, planes=planes,
                            perturb=perturb)
    w = _weighted(_weights(cam["H"], cam["W"], cuda, t0["keep"], seed=seed), bwd)
    t = scale64.tile_truth(raw, c64, (0.0, 0.0, 0.0), tiles, D=3, aa=aa, f=f, planes=planes, weights=w, perturb=perturb)
    return w, t, raw


def _trainer_checks(label, s, k, t, planes, L):
    """-> (discrete checks, values within the per-pixel gates): radii, the last blended Gaussian of every kept pixel, planes, final T"""
    ok = ~t["offender"]
    keep = ~t["excluded"]
    n = t["n_contrib"][keep]
    disc = dict(radii=bool(torch.equal(k["rad"].long()[ok], t["radii"][ok])),
                last=bool(torch.equal(k["last"].reshape(-1)[t["pix"]][keep], t["last"][keep])))
    kern = dict(color=k["img"].reshape(3, -1), depth=k["dep"].reshape(1, -1), alpha=k["A"].reshape(1, -1),
                normal=k["N"].reshape(3, -1) if k["N"] is not None else None, depth2=k["M"].reshape(1, -1) if k["M"] is not None else None)
    good = True
    for p in planes:
        ref = t[p].reshape(-1, t["pix"].numel())[:, keep]
        e = (kern[p][:, t["pix"]][:, keep].double() - ref).abs().amax(0)
        if p in ("depth", "depth2"):
            e = e / float(ref.abs().max())
        good &= _pixel_errs(label, p, e, n, L)
    e = (k["fT"].reshape(-1)[t["pix"]][keep].double() - (1.0 - t["alpha"][keep])).abs()
    good &= _pixel_errs(label, "final_T", e, n, L)
    return disc, good


def _raw_errs(grads, raw, cand):
    errs = {}
    for key, a in zip(s64.RAW, grads):
        _grad_errs(errs, key, a.reshape(a.shape[0], -1), raw[key].grad.reshape(a.shape[0], -1), cand)
    return errs


def _check_emit_reach(name, t, R, P):
    """emit_scan_kernel's two branches, on the trainer's own pass: blocks of 1024 Gaussians in depth order (cdiv(P, 1024) of them).
    Direct writes: a window of 1024 depth-consecutive Gaussians whose non-tight rectangles (listed whole, so their counts are their
    areas) hold more than 2 EM_STAGE instances contains a block above EM_STAGE. Staged writes: the pass's instance count (num_rendered
    of psb_trainer_debug_state) over the blocks is below EM_STAGE, so some block holds at most EM_STAGE."""
    g, tt = t["geo"], t["tiles_touched"]
    live = g["alive"].nonzero().reshape(-1)
    order = live[torch.argsort(g["zd"][live], stable=True)]
    area = tt[order].double()
    nt = torch.where(area > TIGHT_MAX_AREA, area, torch.zeros_like(area))
    cs = torch.cat([torch.zeros(1, dtype=torch.float64, device=area.device), torch.cumsum(nt, 0)])
    blocks = -(-P // 1024)
    print(f"MEASURED emit reach {name}: blocks {blocks}, instances {R}, widest non-tight window {float((cs[1024:] - cs[:-1024]).max()):.0f}")
    assert blocks >= 33 and R < EM_STAGE * blocks
    assert float((cs[1024:] - cs[:-1024]).max()) > 2 * EM_STAGE


@pytest.mark.parametrize("name,fam,bwd,aa,det,f3d", TR_CASES,
                         ids=[f"{n}-{f}-{b}-{'aa' if a else 'plain'}-{'det' if d else 'default'}{'-f3d' if f3 else ''}" for n, f, b, a, d, f3 in TR_CASES])
def test_trainer_at_scale(cuda, name, fam, bwd, aa, det, f3d):
    """render then backwardPixels(grads=...) with weights on the planes `bwd` names (c colour, d depth, a A, n normal, m depth2): radii,
    the last blended Gaussian and final T of every kept pixel, the rendered planes, and the six raw-parameter gradients"""
    s = _scene(name)
    cam = s["cam"]
    W, H = cam["W"], cam["H"]
    c = syn.device_camera(cam, cuda)
    m, tr, f = _trainer(s, cuda, aa, det, f3d, c)
    k = _render(tr, c, fam, bwd, cuda)
    raw0 = s64.raw64(s["sc"], cuda)
    tiles = _trainer_tiles(s, cam, c, aa, raw0, f, cuda)
    planes = _planes(fam, bwd)
    w, t, raw = _truths(s, cam, cuda, tiles, aa, f, planes, bwd)
    grads = [torch.zeros_like(x) for x in m.tensors()]
    tr.backwardPixels(w["color"], w.get("depth"), w.get("alpha"), grads=grads, dL_dnormal=w.get("normal"), dL_ddepth2=w.get("depth2"))
    tr.result()
    torch.cuda.synchronize()
    label = f"trainer {name} {fam} {bwd} aa={aa} det={det} f3d={f3d}"
    bounded = _bound(name, t, max(W, H))
    if s["edge"] == "sky":
        _check_emit_reach(name, t, k["R"], m.num_points())
    disc, good = _trainer_checks(label, s, k, t, planes, max(W, H))
    if s["edge"] == "deep":
        assert int(t["n_contrib"][~t["excluded"]].max()) > 2000
    errs = _raw_errs(grads, raw, t["cand"])
    print(f"MEASURED {label} {errs}")
    assert all(disc.values()), disc
    assert bounded, "exclusions over their bound"
    assert good, "a per-pixel value over its gate"
    _assert_grads(errs)


# Adam mode: one step against step64.adam64 on the truth's gradients. Moments are seeded on every candidate row and on a random half of
# the others, at the size of the group's largest gradient so that every reached element's update is well conditioned.
GATE_ADAM_STEP = 2e-5     # max (|kernel - truth| - one float32 spacing of the parameter) / lr: measured 2.1e-6 (B, opacity)
GATE_ACCUM = 1e-4         # xyz_gradient_accum: max element error / max element: measured 1.3e-5 (B)
ADAM_CASES = [("B", False), ("deep", True)]


@pytest.mark.parametrize("name,det", ADAM_CASES, ids=[f"{n}-{'det' if d else 'default'}" for n, d in ADAM_CASES])
def test_adam_step_at_scale(cuda, name, det):
    """render(check=True) then backwardPixels(grads=None) from seeded moments on a fresh trainer: reached rows against a float64 Adam
    step of the truth's gradients, idle rows (no gradient, no moment) bit for bit unchanged, denom and max_radii2D exact on every
    non-offending row, xyz_gradient_accum within GATE_ACCUM. On deep the first pass overflows the initial binning arena (6 P + 65536
    instances), so the step runs after the retry and must still be one step."""
    import math
    s = _scene(name)
    cam = s["cam"]
    W, H = cam["W"], cam["H"]
    c = syn.device_camera(cam, cuda)
    m, tr, f = _trainer(s, cuda, False, det, False, c)
    P = m.num_points()
    raw0 = s64.raw64(s["sc"], cuda)
    tiles = _trainer_tiles(s, cam, c, False, raw0, f, cuda)
    w, t, raw = _truths(s, cam, cuda, tiles, False, None, _planes("plain", "cda"), "cda")
    gen = torch.Generator(device=cuda).manual_seed(7)
    seeded = torch.rand(P, generator=gen, device=cuda) < 0.5
    seeded[t["cand"]] = True
    for key, ma, va in zip(s64.RAW, m.exp_avg_, m.exp_avg_sq_):
        g = raw[key].grad
        gmax = float(g.abs().max())
        u = lambda: torch.rand(g.shape, generator=gen, device=cuda, dtype=torch.float64)
        sd = seeded.reshape((-1,) + (1,) * (g.dim() - 1)).double()
        ma.copy_(((0.5 * g * (2 * u() - 1) + 0.05 * gmax * (2 * u() - 1)) * sd).float())
        va.copy_(((g * g * (0.5 + u()) + (0.1 * gmax) ** 2) * sd).float())
    m.invalidateAdamLive()
    before = dict(p=[x.detach().double().clone() for x in m.tensors()], m=[x.double().clone() for x in m.exp_avg_],
                  v=[x.double().clone() for x in m.exp_avg_sq_], accum=m.xyz_gradient_accum_.double().clone(), denom=m.denom_.double().clone(),
                  max_radii=m.max_radii2D_.double().clone(), step=m.step_)
    rad = torch.zeros(P, dtype=torch.int32, device=cuda)
    tr.render(c, None, rad, check=True)
    R = _num_rendered(tr, W, H, cuda)
    tr.backwardPixels(w["color"], w["depth"], w["alpha"], grads=None, densify_stats=True)
    tr.result()
    torch.cuda.synchronize()
    if s["edge"] == "deep":
        assert R > 6 * P + 65536, "the view must overflow the initial arena"
    assert m.step_ == before["step"] + 1
    lrs, st = list(m.lr_), before["step"] + 1
    errs = {}
    for i, key in enumerate(s64.RAW):
        g = raw[key].grad
        p1, m1, v1 = step64.adam64(before["p"][i], g, before["m"][i], before["v"][i], lrs[i], st)
        pk = m.tensors()[i].detach()
        rows = lambda x: x.reshape(P, -1)
        idle = (rows(g) == 0).all(1) & (rows(before["m"][i]) == 0).all(1) & (rows(before["v"][i]) == 0).all(1)
        for a, b in ((pk, before["p"][i]), (m.exp_avg_[i], before["m"][i]), (m.exp_avg_sq_[i], before["v"][i])):
            assert torch.equal(rows(a)[idle].double(), rows(b)[idle]), f"an idle row of {key} moved"
        live = ~idle
        ulp = (torch.nextafter(pk, torch.full_like(pk, math.inf)).double() - pk.double()).abs()
        e = ((pk.double() - p1).abs() - ulp).clamp_min(0)
        errs[f"step-{key}"] = float(rows(e)[live].max()) / lrs[i]
        errs[f"grad-m-{key}"] = _relnorm(rows(m.exp_avg_[i])[live], rows(m1)[live])
        errs[f"grad-v-{key}"] = _relnorm(rows(m.exp_avg_sq_[i])[live], rows(v1)[live])
    ok = ~t["offender"]
    vis = t["radii"] > 0
    assert torch.equal(m.denom_.double()[ok], (before["denom"] + vis.double()[:, None])[ok]), "denom"
    mr = torch.where(vis, torch.maximum(before["max_radii"], t["radii"].double()), before["max_radii"])
    assert torch.equal(m.max_radii2D_.double()[ok], mr[ok]), "max_radii2D"
    ndc = t["mean2D_grad"] * torch.tensor([0.5 * W, 0.5 * H], dtype=torch.float64, device=cuda)
    acc = before["accum"] + torch.where(vis, ndc.norm(dim=1), torch.zeros_like(vis, dtype=torch.float64))[:, None]
    errs["accum"] = _maxerr(m.xyz_gradient_accum_, acc, float(acc.abs().max()))
    print(f"MEASURED adam {name} det={det} instances {R} (initial arena {6 * P + 65536}) {errs}")
    for key, v in errs.items():
        gate = GATE_ADAM_STEP if key.startswith("step") else GATE_ACCUM if key == "accum" else GATE_GRAD
        assert v < gate, (key, v, gate)


def test_second_deterministic_pass_against_its_own_truth(cuda):
    """two deterministic passes of one trainer over two views of B (the second shifted by a fraction of the image, so that every tile
    list differs): the second pass's gradients match the second view's truth, so a slot the first pass filled and the second did not
    flush reads as zero (sum_slots skips stale sequence tags)"""
    s = _scene("B")
    cam1 = s["cam"]
    Wc, Hc, fx, fy = syn.CAMERAS["replica"]
    cam2 = syn.make_camera(Wc, Hc, fx, fy, None, np.array([0.07, -0.04, 0.0]))
    c1, c2 = syn.device_camera(cam1, cuda), syn.device_camera(cam2, cuda)
    m, tr, _ = _trainer(s, cuda, False, True, False, c1)
    raw0 = s64.raw64(s["sc"], cuda)
    for cam, c, seed in ((cam1, c1, 1), (cam2, c2, 2)):
        k = _render(tr, c, "plain", "cda", cuda)
        tiles = _trainer_tiles(s, cam, c, False, raw0, None, cuda)
        w, t, raw = _truths(s, cam, cuda, tiles, False, None, _planes("plain", "cda"), "cda", seed=seed)
        grads = [torch.zeros_like(x) for x in m.tensors()]
        tr.backwardPixels(w["color"], w["depth"], w["alpha"], grads=grads)
        tr.result()
        torch.cuda.synchronize()
    disc, good = _trainer_checks("trainer B second view", s, k, t, _planes("plain", "cda"), max(cam2["W"], cam2["H"]))
    errs = _raw_errs(grads, raw, t["cand"])
    print(f"MEASURED second deterministic pass {errs}")
    assert all(disc.values()) and good
    _assert_grads(errs)


# ---- the gates bite -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("what", ["drop", "swap", "truncate"])
def test_perturbed_truth_fails_the_gates(cuda, what):
    """against the deep scene's operator pass: the first contributor of a pixel dropped from its tile's list, the first two
    contributors of a pixel (adjacent in its depth order) swapped, every list cut after 4096 entries. The discrete gates (list
    lengths, contributor counts) or the per-pixel value gates must reject each."""
    s = _scene("deep")
    _, tiles, t0, _, k = _op_pass(cuda, "deep", False)
    W = s["cam"]["W"]
    g = t0["geo"]
    ti = tiles.index((37, 21))
    if what == "truncate":
        perturb = dict(truncate=4096)
    else:
        # a kept pixel of a bench tile: its first contributors blend at T near 1, so one of them dropped or two swapped moves it far
        px = int((~t0["excluded"] & (t0["n_contrib"] >= 5) & (t0["tile"] != ti)).nonzero()[0])
        ti = int(t0["tile"][px])
        tx, ty = tiles[ti]
        r = g["rect"]
        lst = (g["alive"] & (r[:, 0] <= tx) & (tx < r[:, 2]) & (r[:, 1] <= ty) & (ty < r[:, 3])).nonzero().reshape(-1)
        lst = lst[torch.argsort(g["zd"][lst], stable=True)]
        p = int(t0["pix"][px])
        dx, dy = g["means2D"][lst, 0] - float(p % W), g["means2D"][lst, 1] - float(p // W)
        cn = g["conic"][lst]
        a = g["o"][lst] * torch.exp(-0.5 * (cn[:, 0] * dx * dx + cn[:, 2] * dy * dy) - cn[:, 1] * dx * dy)
        contrib = lst[a >= 1.0 / 255.0]
        perturb = dict(drop=(ti, int(contrib[0]))) if what == "drop" else dict(swap=(ti, int(contrib[0]), int(contrib[1])))
    _, _, t, _, _ = _op_pass(cuda, "deep", False, perturb=perturb)
    disc, pix = _op_errs("deep", s, tiles, t, k)
    keep = ~t["excluded"]
    val_ok = all((e <= _pix_gate(max(s["cam"]["W"], s["cam"]["H"]), n)).all() for e, n in pix.values())
    print(f"MEASURED perturbed {what}: discrete {disc}, values within gate {val_ok}, kept pixels {int(keep.sum())}")
    assert not val_ok, f"{what}: the per-pixel value gates do not see the perturbation"
    if what == "truncate":
        assert not disc["list_len"], "the list-length gate does not see the truncation"


def test_perturbed_truth_fails_the_trainer_gates(cuda):
    """the trainer's gates against a truth with the first contributor of a kept pixel dropped from its list: the last blended Gaussian or
    the per-pixel values, and the gradient gates, must each reject it"""
    s = _scene("B")
    cam = s["cam"]
    c = syn.device_camera(cam, cuda)
    m, tr, _ = _trainer(s, cuda, False, False, False, c)
    k = _render(tr, c, "plain", "cda", cuda)
    raw0 = s64.raw64(s["sc"], cuda)
    tiles = _trainer_tiles(s, cam, c, False, raw0, None, cuda)
    _, t0, _ = _truths(s, cam, cuda, tiles, False, None, _planes("plain", "cda"), "cda")
    px = int((~t0["excluded"] & (t0["n_contrib"] >= 5)).nonzero()[0])
    ti = int(t0["tile"][px])
    g = t0["geo"]
    tx, ty = tiles[ti]
    r = g["rect"]
    lst = (g["alive"] & (r[:, 0] <= tx) & (tx < r[:, 2]) & (r[:, 1] <= ty) & (ty < r[:, 3])).nonzero().reshape(-1)
    lst = lst[torch.argsort(g["zd"][lst], stable=True)]
    p = int(t0["pix"][px])
    dx, dy = g["means2D"][lst, 0] - float(p % cam["W"]), g["means2D"][lst, 1] - float(p // cam["W"])
    cn = g["conic"][lst]
    a = g["o"][lst] * torch.exp(-0.5 * (cn[:, 0] * dx * dx + cn[:, 2] * dy * dy) - cn[:, 1] * dx * dy)
    gid = int(lst[a >= 1.0 / 255.0][0])
    w, t, raw = _truths(s, cam, cuda, tiles, False, None, _planes("plain", "cda"), "cda", perturb=dict(drop=(ti, gid)))
    grads = [torch.zeros_like(x) for x in m.tensors()]
    tr.backwardPixels(w["color"], w["depth"], w["alpha"], grads=grads)
    tr.result()
    torch.cuda.synchronize()
    disc, good = _trainer_checks("trainer perturbed drop", s, k, t, _planes("plain", "cda"), max(cam["W"], cam["H"]))
    errs = _raw_errs(grads, raw, t["cand"])
    print(f"MEASURED perturbed trainer drop: discrete {disc}, values within gate {good}, {errs}")
    assert not (disc["last"] and good), "the per-pixel gates do not see the perturbation"
    assert any(v > (GATE_GRAD if key.startswith("grad-") else GATE_GRAD_MAX) for key, v in errs.items()), "the gradient gates do not see it"
