"""Host-side logic of the keyframe-sharded data-parallel path (SURVEY.md §8e). Device-agnostic (torch tensors on
any device, any torch.distributed backend): exercised with gloo on CPU in tests/test_parallel_cpu.py and with NCCL
on the GPUs by trainer.DataParallelTrainer / bench.py --gpus N."""
import torch

SIZES = (3, 3, 45, 1, 3, 4)   # floats per Gaussian of xyz, features_dc, features_rest, opacity, scaling, rotation (csrc row_floats)
PER_GAUSSIAN = sum(SIZES)     # 59


def row_shapes(P):
    """Shapes of the six tensors of a P-row model: [P, 3], [P, 1, 3], [P, 15, 3], [P, 1], [P, 3], [P, 4] (the SH features per channel)."""
    return [(P, k // 3, 3) if i in (1, 2) else (P, k) for i, k in enumerate(SIZES)]


def shard_schedule(schedule, rank, world):
    """Rank r consumes entries r, r+K, r+2K, ... of the shuffled keyframe schedule: K consecutive entries of the
    reference's single-view schedule (gaussian_mapper.cpp:1126-1173) form one data-parallel step."""
    usable = len(schedule) - len(schedule) % world
    return list(schedule[rank:usable:world])


CHUNK = 128                   # Gaussians per ownership chunk of the NVLink data-parallel step (= one backward block)


def owner_of_rows(P, world, device="cpu"):
    """int64 [P]: rank that owns each Gaussian's optimizer state in the p2p step (psb_dp_*): chunk c = row // 128 belongs
    to rank c % world — interleaved, so the records every rank pushes spread evenly over all NVLink destinations at any
    moment of the backward kernel (contiguous shards would make all ranks hit the same owner at the same time)."""
    return (torch.arange(P, device=device) // CHUNK) % world


def gather_owned_rows(tensors, rank, world, group=None):
    """In place: every tensor [P, ...] ends up with row r taken from the rank that owns r. Implemented as zero the rows of
    other owners + all-reduce(SUM) — rare (before densification / a checkpoint), any backend."""
    import torch.distributed as dist
    if world == 1:
        return
    for t in tensors:
        mine = (owner_of_rows(t.size(0), world, t.device) == rank).view(-1, *([1] * (t.dim() - 1)))
        t.mul_(mine.to(t.dtype))
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)


def _pad4(n):
    return -(-n // 4) * 4


class GradBuffer:
    """ONE flat float32 buffer with six views in the reference's tensor shapes, so the whole gradient of a step is a single
    all-reduce call. Every segment starts on a 16-byte boundary (the kernels store the features_rest and rotation gradients
    with 128-bit accesses; P need not be a multiple of 4): [P*59 (+ up to 3 pad floats per segment)]."""

    def __init__(self, P, device):
        self.P = P
        self.flat = torch.zeros(sum(_pad4(P * s) for s in SIZES), dtype=torch.float32, device=device)
        self.segments, o = [], 0
        for s in SIZES:
            self.segments.append(self.flat[o:o + P * s])
            o += _pad4(P * s)

    def views(self):
        return [seg.view(*sh) for seg, sh in zip(self.segments, row_shapes(self.P))]

    def all_reduce(self, group=None):
        """Sum over ranks; returns the factor the optimizer applies (mean over the K views of the step)."""
        import torch.distributed as dist
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        if world > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group)
        return 1.0 / world


def reduce_densify_stats(max_radii2D, xyz_gradient_accum, denom, group=None):
    """Called once, right before densify/prune: max over ranks for the radii, sum for the accumulators
    (every rank then holds the statistics of all views seen since the last densification)."""
    import torch.distributed as dist
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(max_radii2D, op=dist.ReduceOp.MAX, group=group)
        dist.all_reduce(xyz_gradient_accum, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(denom, op=dist.ReduceOp.SUM, group=group)


class SlabGradBuffer:
    """The same [P*59] floats, laid out slab-major: Gaussians are cut into `nslabs` contiguous ranges (boundaries at
    multiples of 128) and each slab keeps its six gradient blocks back to back, so ONE all-reduce call per slab covers
    all parameters of those Gaussians and can start as soon as the slab's backward kernel has finished."""

    def __init__(self, P, device, nslabs=4):
        self.P = P
        per = -(-P // nslabs)
        per = -(-per // 128) * 128
        self.slabs = []           # (first, count)
        f = 0
        while f < P:
            self.slabs.append((f, min(per, P - f)))
            f += per
        self.flat = torch.zeros(max(sum(self._slab_floats(c) for _, c in self.slabs), 4), dtype=torch.float32, device=device)

    def _slab_floats(self, count):
        return sum(_pad4(count * k) for k in SIZES)

    def region(self, s):
        o = sum(self._slab_floats(c) for _, c in self.slabs[:s])
        return self.flat[o:o + self._slab_floats(self.slabs[s][1])]

    def blocks(self, s):
        """Six 1-D views (one per parameter tensor) of slab s, each starting on a 16-byte boundary."""
        first, count = self.slabs[s]
        out, o = [], sum(self._slab_floats(c) for _, c in self.slabs[:s])
        for k in SIZES:
            out.append(self.flat[o:o + count * k])
            o += _pad4(count * k)
        return out

    def kernel_pointers(self, s):
        """Base addresses such that row g of tensor i lands at blocks(s)[i][(g - first) * SIZES[i]] (see psb_trainer_backward_slab)."""
        first, _ = self.slabs[s]
        return [b.data_ptr() - first * k * 4 for b, k in zip(self.blocks(s), SIZES)]


# ------------------------------------------------------------------------------------------------------------------------
# Host-side specification of the record protocol of the NVLink data-parallel step (csrc/psb_train.cu:
# gaussian_backward_kernel<PUSH>, shard_adam_small_kernel; DESIGN.md §8). Device-agnostic torch code: the CPU / gloo test
# tests/test_parallel_cpu.py runs the whole step with it (per-rank gradients from the C oracle), and it documents what the
# kernels exchange: per Gaussian that received a gradient, ONE 80-byte record
#     [ g_xyz 3 | g_f_dc 3 | g_opacity 1 | g_scaling 3 | g_rotation 4 | masked dL/dRGB 3 | pad 2 | epoch ]
# The 45 f_rest gradients are not sent: they are the rank-1 product  w_k(dir) * dL/dRGB[ch]  (reference backward.cu:20-139), and
# the owner re-evaluates w_k from its own copy of xyz and the sender's camera centre.
# ------------------------------------------------------------------------------------------------------------------------
REC_FLOATS = 20
_SH_C0 = 0.28209479177387814
_SH_C1 = 0.4886025119029199
_SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
_SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658, 1.445305721320277,
          -0.5900435899266435)


def sh_basis_weights(xyz, campos, degree):
    """[P, 16] weights dRGB/dsh_k of the real SH basis along normalize(xyz - campos); columns beyond (degree+1)^2 are zero."""
    d = xyz - campos.reshape(1, 3)
    d = d / torch.sqrt((d * d).sum(dim=1, keepdim=True))
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    w = [torch.full_like(x, _SH_C0), -_SH_C1 * y, _SH_C1 * z, -_SH_C1 * x,
         _SH_C2[0] * xy, _SH_C2[1] * yz, _SH_C2[2] * (2.0 * zz - xx - yy), _SH_C2[3] * xz, _SH_C2[4] * (xx - yy),
         _SH_C3[0] * y * (3.0 * xx - yy), _SH_C3[1] * xy * z, _SH_C3[2] * y * (4.0 * zz - xx - yy), _SH_C3[3] * z * (2.0 * zz - 3.0 * xx - 3.0 * yy),
         _SH_C3[4] * x * (4.0 * zz - xx - yy), _SH_C3[5] * z * (xx - yy), _SH_C3[6] * x * (xx - 3.0 * yy)]
    w = torch.stack(w, dim=1)
    w[:, (degree + 1) ** 2:] = 0.0
    return w


def pack_records(grads, masked_drgb, epoch):
    """grads: the six raw-parameter gradients of ONE view (reference shapes; features_rest is ignored), masked_drgb [P,3] = clamp-masked
    dL/dRGB. -> [P, 20] float32 records; rows without any gradient carry epoch 0 (= not sent)."""
    P = grads[0].size(0)
    rec = torch.zeros((P, REC_FLOATS), dtype=torch.float32, device=grads[0].device)
    rec[:, 0:3], rec[:, 3:6], rec[:, 6:7] = grads[0], grads[1].reshape(P, 3), grads[3].reshape(P, 1)
    rec[:, 7:10], rec[:, 10:14], rec[:, 14:17] = grads[4], grads[5], masked_drgb
    sends = rec[:, :17].abs().sum(dim=1) > 0
    rec[:, 19] = torch.where(sends, torch.full((P,), float(epoch)), torch.zeros(P)).to(rec.device)
    return rec


def reduce_records(records, xyz, campos_all, degree, epoch):
    """Owner side: records = [world][P_owned, 20] of the rows this rank owns, xyz [P_owned, 3], campos_all [world, 3].
    -> the six summed raw-parameter gradients of those rows (features_rest reconstructed from the basis weights)."""
    n = xyz.size(0)
    acc = torch.zeros((n, 14), dtype=torch.float32, device=xyz.device)
    g_rest = torch.zeros((n, 15, 3), dtype=torch.float32, device=xyz.device)
    for s, rec in enumerate(records):
        live = (rec[:, 19] == float(epoch)).unsqueeze(1).float()      # stale epoch word: rank s sent nothing for that row
        acc += rec[:, :14] * live
        w = sh_basis_weights(xyz, campos_all[s], degree)[:, 1:]       # [n, 15]
        g_rest += w.unsqueeze(2) * (rec[:, 14:17] * live).unsqueeze(1)
    return [acc[:, 0:3], acc[:, 3:6].reshape(n, 1, 3), g_rest, acc[:, 6:7], acc[:, 7:10], acc[:, 10:14]]
