"""Image-batch data parallelism for the GS-SDF step (SURVEY.md section 8e): splat/SDF state replicated, rank r renders its
own camera, ONE all-reduce of the flat gradient per step, densification statistics reduced so that every replica makes
identical grow/prune decisions. torch.distributed is plumbing (NCCL over NVLink on GPUs, gloo in the CPU tests).

Reference behaviour being parallelised: one image per step drawn from a per-epoch torch::randperm(train_num)
(include/neural_mapping/neural_mapping.cpp:208-225); densification state grad2d/count (sum) and vis/radii (max)
(include/neural_gaussian/neural_gaussian.cpp:660-679).
"""
import torch
import torch.distributed as dist


def epoch_permutation(n_train, epoch, seed=0):
    """Rank-shared permutation of the training images for one epoch (same generator seed on every rank)."""
    g = torch.Generator(device="cpu").manual_seed(seed * 1_000_003 + epoch)
    return torch.randperm(n_train, generator=g)


def image_for_rank(step, rank, world, n_train, seed=0):
    """Image index rank `rank` renders at global step `step`: perm[(step * world + rank) mod n_train] of the epoch's permutation.
    Within an epoch no image is rendered twice and ranks never collide (world <= n_train)."""
    per_epoch = max(n_train // world, 1)
    epoch, i = divmod(step, per_epoch)
    perm = epoch_permutation(n_train, epoch, seed)
    return int(perm[(i * world + rank) % n_train])


def allreduce_flat_grad(flat_grad, world=None, average=True):
    """Sum (or mean) the flat gradient buffer over ranks in place: the path's only data exchange."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return flat_grad
    dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM)
    if average:
        flat_grad.div_(world or dist.get_world_size())
    return flat_grad


def allreduce_densify_state(state):
    """state: dict with 'grad2d', 'count' (summed over ranks) and 'vis', 'radii' (max over ranks); in place."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return state
    for k in ("grad2d", "count"):
        if k in state:
            dist.all_reduce(state[k], op=dist.ReduceOp.SUM)
    for k in ("vis", "radii"):
        if k in state:
            dist.all_reduce(state[k], op=dist.ReduceOp.MAX)
    return state


class GradientExchange:
    """The step's two all-reduces, each overlapped with compute that does not depend on it (DESIGN.md section 8):

        sdf segment   (hash table + decoder): final after stage [C]  -> reduced under the render backward [D] of the same step
        splat segment                        : final after [D]        -> reduced under stage [A] of the NEXT step (which reads SDF
                                               parameters only); `before_render` waits for it before the splats are touched again

    Plug the three methods into GsSdfStep.step(on_sdf_grads_ready=..., before_render=...) and call finish_step() after it; drain()
    before reading the gradients / stopping a timer. Works with any torch.distributed backend (NCCL on GPUs, gloo in the CPU tests);
    a no-op when torch.distributed is not initialised or the world size is 1."""

    def __init__(self):
        self.active = dist.is_initialized() and dist.get_world_size() > 1
        self._sdf, self._splat = [], []

    def on_sdf_grads_ready(self, sdf_segment):
        if self.active:
            self._sdf.append(dist.all_reduce(sdf_segment, op=dist.ReduceOp.SUM, async_op=True))

    def before_render(self):
        while self._splat:
            self._splat.pop().wait()

    def finish_step(self, splat_segment):
        """splat_segment None: the caller exchanges the splat gradient itself (SparseRowExchange)"""
        if not self.active:
            return
        if splat_segment is not None:
            self._splat.append(dist.all_reduce(splat_segment, op=dist.ReduceOp.SUM, async_op=True))
        while self._sdf:
            self._sdf.pop().wait()

    def drain(self):
        self.before_render()
        while self._sdf:
            self._sdf.pop().wait()


class SparseRowExchange:
    """Exchange of the splat-gradient segment by its VISIBLE rows (CUDA trainers, one camera per rank and step). Only the rows of the
    splats a rank's frame sees carry a gradient, so instead of all-reducing the dense [N x 59] segment the ranks all-gather

        packed[k] = [row id | offsets | quaternion | scaling | opacity | features_dc | features_rest]   k < nnz(rank)

    (gssdf_rows_pack, which also clears those rows locally) and every rank adds ALL ranks' packed rows, its own included, in rank order
    (gssdf_rows_unpack_add): the same sum on every rank, bit for bit, like after an all-reduce. The row counts differ per rank and step;
    they are exchanged first (one int32 per rank), read on the host while the render backward is still queued on the device, and the
    all-gather is sized to the largest count. use_sparse() falls back to the dense all-reduce unless the gathered rows are less than half
    the dense segment (larger world sizes, most splats visible)."""

    def __init__(self, trainer, world, rank, always=False):
        from . import cabi
        self.always = always
        self.cabi, self.T, self.world, self.rank = cabi, trainer, world, rank
        N = trainer.N_cap
        self.segments = [(trainer.seg_off[i], trainer.seg_w[i]) for i in range(6) if trainer.seg_w[i] > 0]
        self.stride = cabi.rows_stride(self.segments)
        dev = trainer.flat_grad.device
        self.cnt_all = torch.zeros(world, dtype=torch.int32, device=dev)
        self.cnt_host = torch.zeros(world, dtype=torch.int32).pin_memory()
        self.cnt_ev = torch.cuda.Event()
        self.dense_bytes = trainer.t0 * 4
        self.pack = self.gath = None
        self.rows = 0
        self._N = N

    def start_counts(self):
        """enqueue: all-gather of the ranks' visible-row counts -> pinned host (call once the step's projection has been enqueued)"""
        dist.all_gather_into_tensor(self.cnt_all, self.T.R.counts[0:1])
        self.cnt_host.copy_(self.cnt_all, non_blocking=True)
        self.cnt_ev.record()

    def use_sparse(self):
        """host: wait for the counts (the device still has the render backward queued) and size this step's exchange"""
        self.cnt_ev.synchronize()
        rows = (int(self.cnt_host.max()) + 255) // 256 * 256
        self.rows = min(max(rows, 256), self._N)
        # the row exchange saves wire time but adds pack / unpack launches and a host read of the counts: sparse only while the
        # gathered rows are clearly smaller than the dense segment
        return self.always or self.world * self.rows * self.stride * 4 <= 0.5 * self.dense_bytes

    def launch(self):
        T, rows, st = self.T, self.rows, self.stride
        if self.pack is None or self.pack.numel() < rows * st:
            cap = min(int(rows * 1.25), self._N)
            self.pack = torch.empty(cap * st, dtype=torch.float32, device=T.flat_grad.device)
            self.gath = torch.empty(self.world * cap * st, dtype=torch.float32, device=T.flat_grad.device)
        self.cabi.rows_pack(self.segments, rows, T.R.counts[0:1], T.R.p["gaussian_ids"], T.flat_grad, self.pack, zero_source=True)
        return dist.all_gather_into_tensor(self.gath[:self.world * rows * st], self.pack[:rows * st], async_op=True)

    def add_all(self):
        rows, st = self.rows, self.stride
        for p in range(self.world):  # rank order on every rank: identical sums
            self.cabi.rows_unpack_add(self.segments, rows, self.cnt_all[p:p + 1], self.T.flat_grad, self.gath[p * rows * st:(p + 1) * rows * st])


class DataParallelStep:
    """One data-parallel training step around a trainer object (render.GsSdfTrainer, or any object with the same five members):

        trainer.train_step(*args, on_sdf_grads_ready=..., before_render=..., **kw)   writes the flat gradient [splat segment | SDF segment]
        trainer.flat_grad, trainer.t0                                               t0 = first element of the SDF segment
        trainer.adam_sdf(grad_scale), trainer.adam_splat(grad_scale), trainer.adam_all(grad_scale)

    Single process: train_step then adam_all. world > 1: the two all-reduces of GradientExchange, and each segment's Adam update (with
    grad_scale = 1 / world: the reduced gradient is a sum of per-rank means) as soon as its reduction is complete -- SDF groups right
    after the step, splat groups just before the next render touches the splats (the splat all-reduce runs under the next step's
    sample generation + SDF stage). Every rank applies the same update to its replica. Call flush() before reading parameters or
    stopping a timer: it completes the last step's splat update."""

    def __init__(self, trainer, world=None, sparse_rows=True):
        """sparse_rows: True = exchange the splat segment by its visible rows when the gathered rows are less than half the dense segment (CUDA
        trainers with one camera per step; see SparseRowExchange), "always" = whenever possible, False = dense all-reduce only."""
        self.T = trainer
        self.world = world if world is not None else (dist.get_world_size() if dist.is_initialized() else 1)
        self.x = GradientExchange()
        self._pending_splat = False
        self.sparse = None
        fg = getattr(trainer, "flat_grad", None)
        if (sparse_rows and self.world > 1 and dist.is_initialized() and fg is not None and fg.is_cuda and hasattr(trainer, "seg_off")
                and getattr(getattr(trainer, "R", None), "C", 0) == 1):
            self.sparse = SparseRowExchange(trainer, self.world, dist.get_rank(), always=(sparse_rows == "always"))
        self._sparse_work = None
        self.sparse_steps = self.dense_steps = 0
        self.cover_dense_exchange = True

    def _mark(self, name):
        R = getattr(self.T, "R", None)
        if R is not None and hasattr(R, "_mark"):
            R._mark(name)  # profiling hook of the renderer (bench.py's per-stage table); no-op unless enabled

    def _before_render(self):
        self.x.before_render()
        if self._sparse_work is not None:
            self._sparse_work.wait()
            self._sparse_work = None
            self.sparse.add_all()
        self._mark("wait_splat_allreduce")
        if self._pending_splat:
            self.T.adam_splat(1.0 / self.world)
            self._pending_splat = False

    def step(self, *args, **kw):
        T = self.T
        if self.world <= 1:
            out = T.train_step(*args, **kw)
            T.adam_all(1.0)
            return out
        out = T.train_step(*args, on_sdf_grads_ready=self._on_sdf_grads_ready, before_render=self._before_render, **kw)
        if self.sparse is not None and self.sparse.use_sparse():
            self._sparse_work = self.sparse.launch()  # visible rows in flight
            self.x.finish_step(None)                  # returns once the SDF segment is reduced
            self.sparse_steps += 1
        else:
            self.x.finish_step(T.flat_grad[:T.t0])  # splat all-reduce in flight; returns once the SDF segment is reduced
            self.dense_steps += 1
        self._mark("wait_sdf_allreduce")
        if self.cover_dense_exchange and hasattr(T, "overlap_ray_stage"):
            # two-stream schedule: with the dense all-reduce in flight the next step's sample generation + [A] stay on the caller's stream,
            # ahead of the wait for it; with the (short) row exchange they go to the second stream like on a single GPU
            T.overlap_ray_stage = self._sparse_work is not None
        self._pending_splat = True
        T.adam_sdf(1.0 / self.world)
        return out

    def _on_sdf_grads_ready(self, sdf_segment):
        self.x.on_sdf_grads_ready(sdf_segment)
        if self.sparse is not None:
            self.sparse.start_counts()

    def flush(self):
        if self.world > 1:
            self._before_render()
