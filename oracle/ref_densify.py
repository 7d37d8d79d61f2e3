"""TEST INFRASTRUCTURE ONLY — GaussianModel::densifyAndPrune and friends restated op for op with the ATen ops the reference's
LibTorch code calls (reference src/gaussian_model.cpp:556-815; include/general_utils.h:25-56). Works on CPU or CUDA tensors.

It pins oracle/gs_oracle.c:orc_densify_and_prune on CPU (tests/test_oracle_cpu.py) and checks the fused CUDA kernel
(psb_densify_*) on the GPU (tests/test_densify_gpu.py). The one random op, at::normal(means, stds) (:734), is replaced by
`means + stds * z` with an injected z so that all three implementations see the same draw.

state = dict(p=[6 tensors], m=[6], v=[6], accum=[P,1], denom=[P,1], max_radii=[P])   (reference tensor shapes)
"""
import torch


def _sig(x): return torch.sigmoid(x)                      # getOpacityActivation
def _exp(x): return torch.exp(x)                          # getScalingActivation


def build_rotation(r):
    """include/general_utils.h:31-56"""
    r0, r1, r2, r3 = r[:, 0], r[:, 1], r[:, 2], r[:, 3]
    norm = torch.sqrt(r0 * r0 + r1 * r1 + r2 * r2 + r3 * r3)
    q = r / norm.unsqueeze(1)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.zeros((q.size(0), 3, 3), dtype=r.dtype, device=r.device)
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - w * z); R[:, 0, 2] = 2 * (x * z + w * y)
    R[:, 1, 0] = 2 * (x * y + w * z); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - w * x)
    R[:, 2, 0] = 2 * (x * z - w * y); R[:, 2, 1] = 2 * (y * z + w * x); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def prune_points(st, mask):
    """:588-642"""
    valid = ~mask
    for key in ("p", "m", "v"):
        st[key] = [t[valid].clone() for t in st[key]]
    st["accum"], st["denom"], st["max_radii"] = st["accum"][valid], st["denom"][valid], st["max_radii"][valid]


def densification_postfix(st, ext):
    """:644-714: parameters concatenated, moments zero-extended, statistics reset"""
    st["p"] = [torch.cat((t, e), dim=0) for t, e in zip(st["p"], ext)]
    st["m"] = [torch.cat((t.clone(), torch.zeros_like(e)), dim=0) for t, e in zip(st["m"], ext)]
    st["v"] = [torch.cat((t.clone(), torch.zeros_like(e)), dim=0) for t, e in zip(st["v"], ext)]
    P, dev = st["p"][0].size(0), st["p"][0].device
    st["accum"], st["denom"], st["max_radii"] = torch.zeros((P, 1), device=dev), torch.zeros((P, 1), device=dev), torch.zeros(P, device=dev)


def densify_and_clone(st, grads, grad_threshold, scene_extent, percent_dense):
    """:763-793"""
    sel = torch.where(torch.linalg.vector_norm(grads, dim=-1) >= grad_threshold, True, False)
    sel = torch.logical_and(sel, torch.max(_exp(st["p"][4]), dim=1).values <= percent_dense * scene_extent)
    densification_postfix(st, [t[sel] for t in st["p"]])
    return int(sel.sum())


def densify_and_split(st, grads, grad_threshold, scene_extent, percent_dense, z, N=2):
    """:716-761; z: [N * n_selected, 3] standard-normal draw (None -> torch.randn)"""
    n_init = st["p"][0].size(0)
    dev = st["p"][0].device
    padded = torch.zeros(n_init, dtype=grads.dtype, device=dev)
    padded[:grads.size(0)] = grads.squeeze()
    sel = torch.where(padded >= grad_threshold, True, False)
    sel = torch.logical_and(sel, torch.max(_exp(st["p"][4]), dim=1).values > percent_dense * scene_extent)
    stds = _exp(st["p"][4])[sel].repeat(N, 1)
    means = torch.zeros((stds.size(0), 3), device=dev)
    zz = torch.randn_like(stds) if z is None else z.to(dev)
    samples = means + stds * zz                                     # at::normal(means, stds)
    rots = build_rotation(st["p"][5][sel]).repeat(N, 1, 1)
    new_xyz = torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + st["p"][0][sel].repeat(N, 1)
    new_scaling = torch.log(_exp(st["p"][4])[sel].repeat(N, 1) / (0.8 * N))
    ext = [new_xyz, st["p"][1][sel].repeat(N, 1, 1), st["p"][2][sel].repeat(N, 1, 1), st["p"][3][sel].repeat(N, 1), new_scaling,
           st["p"][5][sel].repeat(N, 1)]
    densification_postfix(st, ext)
    prune_filter = torch.cat((sel, torch.zeros(N * int(sel.sum().item()), dtype=torch.bool, device=dev)))
    prune_points(st, prune_filter)
    return int(sel.sum())


def split_count(st, max_grad, extent, percent_dense):
    grads = st["accum"] / st["denom"]
    grads[grads.isnan()] = 0.0
    sel = (grads.squeeze(-1) >= max_grad) & (torch.max(_exp(st["p"][4]), dim=1).values > percent_dense * extent)
    return int(sel.sum())


def densify_and_prune(st, max_grad, min_opacity, extent, max_screen_size, percent_dense, z=None):
    """:795-815. Mutates and returns st."""
    grads = st["accum"] / st["denom"]
    grads[grads.isnan()] = 0.0
    densify_and_clone(st, grads, max_grad, extent, percent_dense)
    densify_and_split(st, grads, max_grad, extent, percent_dense, z)
    prune_mask = (_sig(st["p"][3]) < min_opacity).squeeze(-1)
    if max_screen_size:
        big_vs = st["max_radii"] > max_screen_size
        big_ws = torch.max(_exp(st["p"][4]), dim=1).values > 0.1 * extent
        prune_mask = torch.logical_or(torch.logical_or(prune_mask, big_vs), big_ws)
    prune_points(st, prune_mask)
    return st


def reset_opacity(st):
    """:556-565 (the clamp is a no-op: SURVEY §2.2 quirk 9); fresh moments for the opacity group (:576-578)"""
    act = _sig(st["p"][3])
    new = torch.min(act, torch.ones_like(act * 0.01))
    st["p"][3] = torch.log(new / (1 - new))
    st["m"][3] = torch.zeros_like(st["p"][3])
    st["v"][3] = torch.zeros_like(st["p"][3])
    return st
