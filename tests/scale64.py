"""The float64 truth of tests/splat64.py on a sample of tiles: exact on scenes of millions of Gaussians, where a dense render is not
tractable.

Geometry (radius, rectangle, alive, tiles_touched) is evaluated without grad for all P. Only the candidates of the sampled tiles (alive,
rectangle holding the tile) enter a differentiable pass, indexed out of the leaves. Each tile is composited densely by
splat64.composite(tiles=...) and its weighted pixel sum is back-propagated before the next tile, so memory stays per tile and the
gradient of a loss whose per-pixel weights are non-zero only on the sampled tiles is exact. Rows that are no candidate get exactly zero.
The normal plane (normal64.gaussian_normals) and the second depth moment (dist64: the blend of z^2) are the same composite with the
colour replaced, as those modules state them.

Ambiguity. A decision that float32 rounding could take either way is excluded at the smallest sound grain:
  * pair decisions (power closer than splat64.MIN_MARGIN, alpha_min and alpha_max closer than ALPHA_FLOOR), a depth tie between two
    splats of a pixel that pass its alpha test (relative gap below TIE_ULPS ulps of the view depth's magnitude) and the T test exclude
    the pixel. The kernels' T is a product of float32 factors; each
    factor 1 - alpha carries alpha's error (expf, the power and the opacity: T_ULPS ulps bound it with headroom) amplified by
    1 / (1 - alpha), so the T test is ambiguous when its relative margin is below max(MIN_MARGIN, T_ULPS 2^-24 sum_i 1 / (1 - alpha_i)),
    the sum over the factors blended up to the test. This is k n 2^-24 with each factor weighted by its conditioning; for alpha <= 0.5
    it is at most 2 T_ULPS n 2^-24.
  * Gaussian-level decisions (near, det, radius with its lambda clamp, rectangle edge, frustum clamp, colour clamp, anti-aliasing
    floor) exclude the sampled pixels at which that Gaussian's truth alpha reaches (1/255)(1 - MIN_MARGIN) (for radius and rectangle
    edges only in the row or column of tiles at the ambiguous edge, the only lists they can change, whose length and contributor counts
    become ambiguous), and
    drop it from the exact radii and tiles_touched comparisons. Radius and rectangle edges are gated by an estimate of their float32 error, not by a relative
    MIN_MARGIN: at 1200 px a relative 1e-4 of a pixel coordinate is 0.1 px, which would exclude several percent of a large scene for no
    reason, while the kernels' error is a few ulps of the coordinate. A Gaussian just behind the near plane has no truth geometry to
    draw, so tile_truth refuses it: the scene has to be moved off the plane.
"""
import torch

import normal64 as n64
import splat64 as s64
import step64

ULP = 2.0 ** -24
T_ULPS = 16.0          # per blended factor: alpha's float32 relative error in ulps, before its 1 / (1 - alpha) amplification. It is
                       # the conic's error times |power| (see ALPHA_FLOOR): ~1e-5 relative at |power| = 1, about 4 ulps per factor of
                       # |power| ~ 1 at T's crossing (alpha ~ 0.3, power ~ -1 for an opaque splat); with up to 4 ulps more from expf,
                       # the opacity and the product, and a factor 2 for |power| up to 2, 16. The average factor is better (final T
                       # within 1.2e-4 after 2100 factors on deep: ~1 ulp each), but the test is decided by its worst factors
ALPHA_FLOOR = s64.MIN_MARGIN   # relative: the float32 conic is a chain of products (3D covariance, J W, the inverse) good to ~1e-5,
                               # and |power| reaches 5.5 at the 1/255 threshold; 1e-5 let alpha-test flips through on B
TIE_ULPS = 8.0         # ulps of the view depth's magnitude (sum |V_k2 x_k| + |V_32|) that two splats of one pixel may be apart and swap
EDGE_ULPS = 8.0        # ulps of (|pixel coordinate| + image extent + radius) that a float32 mean and rectangle edge may be off by:
                       # three roundings of the homogeneous coordinate, one each of 1 / w, the NDC and the pixel mapping, two of the edge
COLOUR_FLOOR = 1e-5    # |SH colour before the clamp|: a sum of 16 terms of order one in float32
PLANES = ("color", "depth", "alpha", "normal", "depth2")
PAIR_KINDS = ("power", "alpha_min", "alpha_max", "T", "depth_tie")


def _frac(v):
    return (v - torch.round(v)).abs()


def gauss_offenders(geo, cam):
    """-> ({kind: bool [P]}: Gaussians with a decision of their own within float32 reach of its threshold (module docstring),
    bool [P,4]: which rectangle edges (x0, y0, x1, y1) a shape decision leaves ambiguous)"""
    fr, al = geo["front"], geo["alive"]
    det = geo["det"]
    disc = geo["disc"].detach()
    mid = torch.sqrt(disc.clamp_min(0) + det)   # mid^2 = disc + det
    r3 = geo["r3"].detach()
    lam1 = (r3 / 3.0) ** 2
    sq = torch.sqrt(disc.clamp_min(0.1))
    # disc = mid^2 - det cancels in float32: its error is a few ulps of mid^2 + |det|, and sqrt(max(disc, 0.1)) moves by at most
    # err / (2 sqrt(0.1)) or sqrt(err), whichever is smaller; the clamp at 0.1 only matters through the radius it changes
    err_disc = 4.0 * ULP * (mid * mid + det.abs())
    err_lam = 4.0 * ULP * lam1 + torch.minimum(err_disc / (2.0 * sq), torch.sqrt(err_disc))
    err_r3 = 3.0 * err_lam / (2.0 * torch.sqrt(lam1)) + 4.0 * ULP * r3
    out = dict(near=(geo["zd"] - s64.NEAR).abs() / s64.NEAR < s64.MIN_MARGIN)
    out["det"] = fr & (det.abs() / geo["detscale"] < s64.MIN_MARGIN)
    out["radius"] = fr & (_frac(r3) < 4.0 * err_r3)
    e = geo["edges"].detach()
    W, H = cam["W"], cam["H"]
    lim = torch.tensor([geo["gx"], geo["gy"], geo["gx"], geo["gy"]], dtype=torch.float64, device=e.device)
    live_edge = fr[:, None] & (e >= 0) & (e <= lim + 1)
    p = geo["means2D"].detach()
    reach = (p[:, [0, 1, 0, 1]].abs() + max(W, H) + r3[:, None] + s64.TILE) / s64.TILE
    floor = EDGE_ULPS * ULP * reach
    rect_edge = live_edge & (_frac(e) < floor)
    out["rect"] = rect_edge.any(1)
    lims = (s64.FRUSTUM * cam["tanfovx"], s64.FRUSTUM * cam["tanfovy"])
    out["frustum"] = fr & torch.stack([(r.abs() - l).abs() / l < s64.MIN_MARGIN for r, l in zip(geo["ratios"], lims)], 1).any(1)
    out["colour"] = al & (geo["rgb_pre"].abs() < COLOUR_FLOOR).any(1)
    out["aa"] = al & ((geo["ratio"] - s64.MIN_RATIO).abs() / s64.MIN_RATIO < s64.MIN_MARGIN)
    # the edges a shape decision leaves ambiguous: its own, and for a radius one step away every edge within 1/16 tile of an integer
    amb = rect_edge | (out["radius"][:, None] & live_edge & (_frac(e) < 1.0 / s64.TILE + floor))
    return out, amb


def sample_tiles(W, H, n, seed, must=()):
    """n distinct (tx, ty) of a W x H image, seeded, the tiles in `must` first; partial last-column and last-row tiles always join"""
    gx, gy = -(-W // s64.TILE), -(-H // s64.TILE)
    out = list(dict.fromkeys(tuple(map(int, t)) for t in must))
    if W % s64.TILE:
        out.append((gx - 1, (gy - 1) // 2))
    if H % s64.TILE:
        out.append(((gx - 1) // 2, gy - 1))
    out = list(dict.fromkeys(out))
    gen = torch.Generator().manual_seed(seed)
    for k in torch.randperm(gx * gy, generator=gen).tolist():
        if len(out) >= n:
            break
        t = (k % gx, k // gx)
        if t not in out:
            out.append(t)
    return out


def _inputs(g, raw, f):
    if not raw:
        return g
    return step64.splat_inputs(g, step64.Flags(f3d=f is not None), f)


def tile_truth(leaves, cam, bg, tiles, D=3, aa=False, raw=True, f=None, planes=("color", "depth", "alpha"), weights=None, conv=s64.CONV,
               perturb=None, chunk=256):
    """The truth's forward on `tiles` (a list of (tx, ty)) and, with `weights` ({plane: full-image weights}), the gradient of
    sum_plane sum_{kept sampled pixels} weight * plane, accumulated into leaves[k].grad of the leaves that require grad.

    leaves: float64 trainer parameters (raw=True; f = the 3D filter [P] or None) or activated operator inputs (raw=False).
    cam: splat64.camera64(...). planes: any of PLANES (normal needs raw=True).
    perturb: a deliberately wrong truth for the tests that show the gates bite: dict(drop=(tile, gid)) leaves Gaussian gid out of that
    tile's list, dict(swap=(tile, gid_a, gid_b)) exchanges two splats' depth order there, dict(truncate=n) cuts every list after n.

    -> dict over the N sampled pixels, in tile order: pix [N] (y W + x), tile [N] (index into tiles), the planes (color and normal
    [3,N], the others [N]), n_contrib, last (the global index of the last blended Gaussian, -1 = none), stopped, clamped,
    excluded [N] bool, keep [H,W] (the sampled pixels not excluded: the weights the kernel has to see are weights * keep), list_len
    [len(tiles)], mean2D_grad [P,2] (with weights: dL/dmean2D in pixels), list_ambiguous [len(tiles)] (a shape decision may change the list: skip its length and contributor counts);
    for all P radii, tiles_touched, offender [P] bool (Gaussian-level ambiguity), cand (sorted candidate rows);
    counts (exclusions by kind)."""
    W, H = cam["W"], cam["H"]
    dev = next(iter(leaves.values())).device
    perturb = perturb or {}
    with torch.no_grad():
        geo = s64.geometry(_inputs({k: v.detach() for k, v in leaves.items()}, raw, f), cam, D, aa, conv=conv)
    off_kinds, edge_amb = gauss_offenders(geo, cam)
    offender = torch.stack(list(off_kinds.values()), 0).any(0)
    behind = off_kinds["near"] & ~geo["front"]
    rect, alive = geo["rect"], geo["alive"]
    cover = []
    for tx, ty in tiles:
        cover.append((alive & (rect[:, 0] <= tx) & (tx < rect[:, 2]) & (rect[:, 1] <= ty) & (ty < rect[:, 3])).nonzero().reshape(-1))
        near_tile = (rect[:, 0] <= tx + 1) & (tx - 1 < rect[:, 2]) & (rect[:, 1] <= ty + 1) & (ty - 1 < rect[:, 3])
        if bool((behind & near_tile).any()):
            raise ValueError(f"Gaussians {behind.nonzero().reshape(-1).tolist()[:8]} lie on the near plane: move them off it")
    cand = torch.unique(torch.cat(cover)) if cover else torch.zeros(0, dtype=torch.long, device=dev)
    # the float32 view depth is off by a few ulps of sum_k |V_k2 x_k| + |V_32|; over |z| that is at most this factor on the candidates
    xyz = (leaves["xyz"] if raw else leaves["means3D"]).detach()[cand]
    zmag = xyz.abs() @ cam["V"][:3, 2].abs() + cam["V"][3, 2].abs()
    tie_floor = TIE_ULPS * ULP * float((zmag / geo["zd"][cand].abs()).max()) if cand.numel() else 0.0
    pos = torch.full((geo["zd"].numel(),), -1, dtype=torch.long, device=dev)
    pos[cand] = torch.arange(cand.numel(), device=dev)
    need_grad = weights is not None and any(v.requires_grad for v in leaves.values())
    sub = {k: v.detach()[cand].clone().requires_grad_(need_grad and v.requires_grad) for k, v in leaves.items()}
    f_sub = f[cand] if f is not None else None
    m2_sub = torch.zeros((cand.numel(), 2), dtype=torch.float64, device=dev)
    # pixels of the sampled tiles and the Gaussian-level exclusion: alpha of every front offender at every sampled pixel
    pix = []
    for tx, ty in tiles:
        ys, xs = torch.meshgrid(torch.arange(ty * s64.TILE, min(ty * s64.TILE + s64.TILE, H), device=dev),
                                torch.arange(tx * s64.TILE, min(tx * s64.TILE + s64.TILE, W), device=dev), indexing="ij")
        pix.append((ys * W + xs).reshape(-1))
    allpix = torch.cat(pix)
    px, py = (allpix % W).double(), (allpix // W).double()
    # A value decision (near, det, frustum, colour, aa) may change the Gaussian's alpha or colour on every pixel it reaches. A shape
    # decision (radius, rectangle edge) moves an edge e of its rectangle by one tile, so only the row or column of tiles round(e) - 1
    # next to that edge may or may not list the Gaussian. Those tiles' list lengths and contributor counts are ambiguous, and their
    # pixels that the Gaussian reaches are excluded.
    shape = off_kinds["radius"] | off_kinds["rect"]
    value = offender & ~shape
    ptx, pty = (px // s64.TILE).long(), (py // s64.TILE).long()
    tile_ix = torch.tensor(tiles, dtype=torch.long, device=dev).reshape(-1, 2)
    g_excl = torch.zeros(allpix.numel(), dtype=torch.bool, device=dev)
    list_amb = torch.zeros(len(tiles), dtype=torch.bool, device=dev)
    offs = (offender & geo["front"]).nonzero().reshape(-1)
    e_line = torch.round(geo["edges"].detach()).long() - 1

    def ambiguous(o, tx, ty):
        rc, ea, el = rect[o], edge_amb[o], e_line[o]
        span_x = (tx[None, :] >= rc[:, 0:1] - 1) & (tx[None, :] <= rc[:, 2:3])
        span_y = (ty[None, :] >= rc[:, 1:2] - 1) & (ty[None, :] <= rc[:, 3:4])
        on_x = (ea[:, 0:1] & (tx[None, :] == el[:, 0:1])) | (ea[:, 2:3] & (tx[None, :] == el[:, 2:3]))
        on_y = (ea[:, 1:2] & (ty[None, :] == el[:, 1:2])) | (ea[:, 3:4] & (ty[None, :] == el[:, 3:4]))
        return (on_x & span_y) | (on_y & span_x)

    for i in range(0, offs.numel(), chunk):
        o = offs[i:i + chunk]
        dx = geo["means2D"][o, 0].detach()[:, None] - px[None, :]
        dy = geo["means2D"][o, 1].detach()[:, None] - py[None, :]
        con = geo["conic"][o].detach()
        power = -0.5 * (con[:, 0:1] * dx * dx + con[:, 2:3] * dy * dy) - con[:, 1:2] * dx * dy
        a = geo["o"][o].detach()[:, None] * torch.exp(power)
        reach = a >= conv.alpha_min * (1.0 - s64.MIN_MARGIN)
        amb_pix = ambiguous(o, ptx, pty)
        list_amb |= ambiguous(o, tile_ix[:, 0], tile_ix[:, 1]).any(0)
        g_excl |= (reach & (value[o][:, None] | amb_pix)).any(0)
    res = {k: [] for k in ("color", "depth", "alpha", "normal", "depth2", "n_contrib", "last", "stopped", "clamped", "excluded", "tile")}
    counts = {k: 0 for k in PAIR_KINDS}
    list_len = []
    wgt = {k: v.to(dev, torch.float64) for k, v in (weights or {}).items()}
    start = 0
    for ti, (tx, ty) in enumerate(tiles):
        rows = pos[cover[ti]]
        zd = geo["zd"][cover[ti]]
        if "drop" in perturb and perturb["drop"][0] == ti:
            rows = rows[cover[ti] != perturb["drop"][1]]
        if "truncate" in perturb and rows.numel() > perturb["truncate"]:
            rows = rows[torch.argsort(zd, stable=True)[:perturb["truncate"]].sort().values]
        g_t = {k: v[rows] for k, v in sub.items()}
        geo_t = s64.geometry(_inputs(g_t, raw, f_sub[rows] if f_sub is not None else None), cam, D, aa, conv=conv)
        if "swap" in perturb and perturb["swap"][0] == ti:
            a, b = (int((cand[rows] == gid).nonzero()) for gid in perturb["swap"][1:])
            zs = geo_t["zd"].clone()
            zs[a], zs[b] = zs[b].clone(), zs[a].clone()
            geo_t["zd"] = zs
        out = s64.composite(geo_t, W, H, bg, conv, want_margins=True, tiles=[(tx, ty)])
        assert int(out["list_len"][0]) == rows.numel(), "a candidate's rectangle differs between the full and the per-tile geometry"
        list_len.append(rows.numel() + (1 if "drop" in perturb and perturb["drop"][0] == ti else 0))
        npx = out["pix"].numel()
        assert torch.equal(out["pix"], allpix[start:start + npx])
        pmg = out["pix_margins"]
        excl = g_excl[start:start + npx].clone()
        for k in ("power", "alpha_min", "alpha_max"):
            bad = pmg[k] < (s64.MIN_MARGIN if k == "power" else ALPHA_FLOOR)
            counts[k] += int((bad & ~excl).sum())
            excl |= bad
        bad = (pmg["T"] < s64.MIN_MARGIN) | (pmg["T_ulp"] < T_ULPS)
        counts["T"] += int((bad & ~excl).sum())
        excl |= bad
        bad = pmg["depth_tie"] < tie_floor
        counts["depth_tie"] += int((bad & ~excl).sum())
        excl |= bad
        vals = dict(color=out["color"], depth=out["depth"], alpha=out["alpha"])
        if "normal" in planes:
            n = n64.gaussian_normals(g_t, cam)
            vals["normal"] = s64.composite(dict(geo_t, rgb=n), W, H, (0.0, 0.0, 0.0), conv, tiles=[(tx, ty)])["color"]
        if "depth2" in planes:
            z = geo_t["z"]
            m = torch.stack([z * z, torch.zeros_like(z), torch.zeros_like(z)], 1)
            vals["depth2"] = s64.composite(dict(geo_t, rgb=m), W, H, (0.0, 0.0, 0.0), conv, tiles=[(tx, ty)])["color"][0]
        if need_grad:
            keep = (~excl).double()
            p_t = out["pix"]
            loss = 0.0
            for k, w in wgt.items():
                wk = w.reshape(-1, H * W)[:, p_t] * keep
                loss = loss + (vals[k].reshape(-1, npx) * wk).sum()
            if torch.is_tensor(loss) and loss.requires_grad:
                if geo_t["means2D"].requires_grad:
                    geo_t["means2D"].retain_grad()
                loss.backward()
                if geo_t["means2D"].grad is not None:
                    m2_sub.index_add_(0, rows, geo_t["means2D"].grad)
        for k in ("color", "depth", "alpha", "normal", "depth2"):
            if k in vals:
                res[k].append(vals[k].detach())
        last = out["last"]
        res["last"].append(torch.where(last >= 0, cand[rows][last.clamp_min(0)], last))
        for k in ("n_contrib", "stopped", "clamped"):
            res[k].append(out[k])
        res["excluded"].append(excl)
        res["tile"].append(torch.full((npx,), ti, dtype=torch.long, device=dev))
        start += npx
    if need_grad:
        for k, v in leaves.items():
            if v.requires_grad:
                if v.grad is None:
                    v.grad = torch.zeros_like(v)
                if sub[k].grad is not None:
                    v.grad.index_add_(0, cand, sub[k].grad)
    r = {k: (torch.cat(v, -1) if v else None) for k, v in res.items()}
    if need_grad:          # dL/dmean2D in pixels for every row (the densification statistic's input), zero off the candidates
        r["mean2D_grad"] = torch.zeros((geo["zd"].numel(), 2), dtype=torch.float64, device=dev).index_add_(0, cand, m2_sub)
    keep = torch.zeros(H * W, dtype=torch.bool, device=dev)
    keep[allpix[~r["excluded"]]] = True
    counts.update(gauss={k: int(v.sum()) for k, v in off_kinds.items()}, pixel_gauss=int(g_excl.sum()), pixels=int(allpix.numel()),
                  excluded=int(r["excluded"].sum()), offenders=int(offender.sum()), P=int(offender.numel()))
    r.update(pix=allpix, keep=keep.reshape(H, W), list_len=torch.tensor(list_len, device=dev), list_ambiguous=list_amb, radii=geo["radius"],
             tiles_touched=geo["tiles_touched"], offender=offender, cand=cand, counts=counts, geo=geo)
    return r
