"""Multi-GPU SDS step (SURVEY.md 8e): one process per GPU, G ranks = G camera views per step.

    a G-rank step  ==  single-process accumulation of the same G poses' gradients, then one optimizer step.

(The reference has no working multi-GPU path: nerf/utils.py:255-263 is unreachable.)  Two things shard differently:

  * Stable-Diffusion guidance is VIEW-parallel: rank r encodes / denoises view r only (fixed cost per view).
  * The NeRF render is RAY-parallel (`RayParallel`): its cost is proportional to the number of occupied samples, which varies
    3x with the pose (250 k .. 710 k at 128x128), so a view-parallel render makes every step wait for the slowest pose (round 1:
    0.859 weak-scaling efficiency at 8 GPUs, all of it this straggler).  Instead every rank marches every G-th pixel of ALL G
    views -- ~1/G of every view's samples, balanced by construction -- and
        forward : all-gather of the G x G per-view sample counts (device side, between march and field: the reference's loss means
                  run over a view's TOTAL padded sample count), one all-to-all of image / depth / weights_sum fragments to the
                  view's owner (5 floats per ray), one all-reduce of the G x 2 regulariser sums;
        backward: the same all-to-all in reverse with the gradients, one all-gather of the 2 upstream loss gradients per view;
    then the one all-reduce (SUM) of the hash-grid + MLP gradients (`GradientAllReduce`), as before.

The occupancy grid must stay identical on all ranks: `update_extra_state(seed=shared_seed(...))` is run redundantly with a seed
shared by all ranks (same parameters + same jitter -> bit-identical bitfield), so no broadcast is needed.
"""
import os

import torch
import torch.distributed as dist


def init_distributed(backend=None):
    """Reads RANK / LOCAL_RANK / WORLD_SIZE / MASTER_* (torchrun).  Returns (rank, local_rank, world_size)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, local, world


def pose_index(step, rank, world_size):
    """Pose consumed by `rank` at global step `step`: consecutive poses are dealt round-robin, so the union over ranks of a
    G-rank run equals the pose sequence of a single-process run (nerf/provider.py:266 index semantics, incl. index % 4 == 0
    being the fixed front view)."""
    return step * world_size + rank


def rank_seed(base_seed, rank):
    """Per-rank RNG stream for view-dependent draws (march jitter, light direction, timestep, SD noises)."""
    return int(base_seed) + 1000003 * int(rank)


def shared_seed(base_seed, iteration):
    """Seed shared by ALL ranks for state that must stay replicated (density-grid jitter)."""
    return (int(base_seed) * 2654435761 + int(iteration)) % (2 ** 62)


class GradientAllReduce:
    """Flat-bucket all-reduce of the two optimizer groups of NeRFNetwork.get_params (nerf/network_tcnn.py:195-206):
    encoder.params (12 196 240 fp32, reduced in place, no copy) and the 6 MLP tensors (6 532 fp32, packed into one bucket).
    Payload 48.8 MB per step -> ~0.19 ms at NVLink-4 line rate, 450 GB/s per direction (SURVEY.md section 5)."""

    def __init__(self, encoder_params, mlp_params, op="sum"):
        self.encoder_params = encoder_params
        self.mlp_params = list(mlp_params)
        self.op = op
        n = sum(p.numel() for p in self.mlp_params)
        self._bucket = torch.zeros(n, dtype=torch.float32, device=encoder_params.device)

    def __call__(self):
        if not dist.is_initialized() or dist.get_world_size() == 1:
            return
        world = dist.get_world_size()
        if self.encoder_params.grad is None:
            self.encoder_params.grad = torch.zeros_like(self.encoder_params)
        work = dist.all_reduce(self.encoder_params.grad, op=dist.ReduceOp.SUM, async_op=True)
        off = 0
        for p in self.mlp_params:
            g = p.grad if p.grad is not None else torch.zeros_like(p)
            self._bucket[off:off + p.numel()].copy_(g.reshape(-1))
            off += p.numel()
        dist.all_reduce(self._bucket, op=dist.ReduceOp.SUM)
        work.wait()
        off = 0
        for p in self.mlp_params:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
            p.grad.copy_(self._bucket[off:off + p.numel()].view_as(p))
            off += p.numel()
        if self.op == "mean":
            self.encoder_params.grad.div_(world)
            for p in self.mlp_params:
                p.grad.div_(world)


class RayParallel:
    """Collectives of the ray-parallel render.  Pixel dealing: rank r renders pixels p = i * world + r (i = 0 .. HW/world - 1) of
    every view, as batch rows [v * HW/world + i]; rank v owns view v.  Works on NCCL (CUDA tensors, current stream, no host sync)
    and on gloo (CPU tensors: the host logic is tested at world_size 2 without a GPU)."""

    def __init__(self, group=None):
        if not dist.is_initialized():
            raise RuntimeError("RayParallel needs an initialised process group (parallel.init_distributed())")
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)

    def gather_counts(self, my_counts, out):
        """my_counts int32 [world] (this rank's samples of every view) -> out int32 [world(rank), world(view)]"""
        dist.all_gather_into_tensor(out.view(-1), my_counts.contiguous(), group=self.group)
        return out

    def fragments_to_owner(self, packed, n_views):
        """packed [world * rpv, C]: rows [v * rpv + i] = this rank's pixel i*world + rank of view v  ->  [HW, C]: the complete
        row-major image of the view this rank owns."""
        G = self.world
        assert n_views == G and packed.shape[0] % G == 0
        rpv, Cc = packed.shape[0] // G, packed.shape[1]
        recv = torch.empty_like(packed)
        dist.all_to_all_single(recv, packed.contiguous(), group=self.group)        # recv[r * rpv + i] = pixel i*world + r of MY view
        return recv.view(G, rpv, Cc).permute(1, 0, 2).reshape(G * rpv, Cc)

    def owner_to_fragments(self, full, n_views):
        """inverse of fragments_to_owner for the gradients: [HW, C] of my view -> [world * rpv, C] in batch-row order"""
        G = self.world
        assert n_views == G and full.shape[0] % G == 0
        rpv, Cc = full.shape[0] // G, full.shape[1]
        send = full.view(rpv, G, Cc).permute(1, 0, 2).contiguous().view(G * rpv, Cc)     # send[r * rpv + i] = pixel i*world + r
        recv = torch.empty_like(send)
        dist.all_to_all_single(recv, send, group=self.group)                       # recv[v * rpv + i] = grad of my pixel i of view v
        return recv

    def reduce_losses(self, partial):
        """partial [2, world]: this rank's share of every view's (loss_orient, loss_smooth) -> summed over ranks (out of place:
        the input is also an autograd-visible output of the render)"""
        out = partial.clone()
        dist.all_reduce(out, op=dist.ReduceOp.SUM, group=self.group)
        return out

    def gather_loss_grads(self, g):
        """g [2] = upstream gradient of (loss_orient, loss_smooth) of MY view -> [world(view), 2]"""
        out = torch.empty(self.world, 2, dtype=g.dtype, device=g.device)
        dist.all_gather_into_tensor(out.view(-1), g.contiguous(), group=self.group)
        return out


def max_over_ranks(value, device):
    """max of a python float over all ranks (timing rule: report the slowest rank)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())
