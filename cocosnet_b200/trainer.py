"""Pix2PixTrainer with the reference's methods (trainers/pix2pix_trainer.py:13-138).

Data parallelism is re-designed for one process per GPU: every rank holds a
full replica (same seed -> bit-identical init), takes its contiguous slice of
the batch (what DataParallel.scatter does) and the gradients are summed with
ONE bucketed NCCL all-reduce per optimiser step (G+Corr grads on the G step, D
grads on the D step) and divided by the world size -- the reference's
`sum(losses).mean()` over replicas.  No per-step parameter broadcast.

`run_step` is the launch-bound answer for one GPU: the whole G+D iteration (both forwards, both backwards, both
fused-Adam updates: ~12 000 kernel launches, which the Python/ATen dispatcher cannot issue as fast as an H100 retires
them) is captured ONCE into a CUDA graph after a few eager iterations and replayed from static input buffers.
"""
import os

import torch
import torch.distributed as dist

from . import nhwc, util
from .nets import EMA
from .pix2pix_model import Pix2PixModel

_BUCKET_BYTES = 64 << 20


def _world():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def _rank():
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def shard_batch(data, rank=None, world=None):
    """Contiguous equal chunk of every batched entry (DataParallel.scatter semantics)."""
    world = _world() if world is None else world
    rank = _rank() if rank is None else rank
    if world == 1:
        return data
    out = {}
    for k, v in data.items():
        n = len(v)
        assert n % world == 0, "batch %d not divisible by world size %d" % (n, world)
        per = n // world
        out[k] = v[rank * per:(rank + 1) * per]
    return out


def allreduce_grads(params, world=None, async_op=False):
    """Average the gradients across ranks.  NCCL: one grouped launch over the gradient tensors themselves; async_op
    returns the handle to wait() on (the collective then runs on NCCL's stream beside whatever is enqueued next).
    Other backends (gloo, the CPU tests): bucketed, flattened, summed and divided."""
    world = _world() if world is None else world
    if world == 1:
        return None
    grads = [p.grad for p in params if p.grad is not None]
    if not grads:
        return None
    if dist.get_backend() == "nccl":
        # ONE grouped NCCL launch over the gradient tensors themselves (ncclGroupStart / End around per-tensor
        # all-reduces, averaged in the collective): no flatten, no copy-back, no separate division -- and a fixed
        # sequence of device work, so it is captured into the iteration's CUDA graph like any other kernel.
        with dist._coalescing_manager(device=grads[0].device, async_ops=async_op) as cm:
            for g in grads:
                dist.all_reduce(g, op=dist.ReduceOp.AVG)
        return cm if async_op else None
    buckets, cur, size = [], [], 0
    for g in grads:
        cur.append(g)
        size += g.numel() * g.element_size()
        if size >= _BUCKET_BYTES:
            buckets.append(cur)
            cur, size = [], 0
    if cur:
        buckets.append(cur)
    works = []
    for b in buckets:
        flat = torch.cat([g.reshape(-1) for g in b])
        works.append((dist.all_reduce(flat, op=dist.ReduceOp.SUM, async_op=True), flat, b))
    for work, flat, b in works:
        work.wait()
        flat.div_(world)
        off = 0
        for g in b:
            n = g.numel()
            g.copy_(flat[off:off + n].view_as(g))
            off += n
    return None


class Pix2PixTrainer:
    def __init__(self, opt, resume_epoch=0):
        self.opt = opt
        self.pix2pix_model = Pix2PixModel(opt)
        if len(opt.gpu_ids) > 0:
            self.pix2pix_model.cuda()
            # fixed shapes every step: let cuDNN pick its fastest algorithms
            torch.backends.cudnn.benchmark = not getattr(opt, "no_cudnn_benchmark", False)
            if getattr(opt, "channels_last", False):  # NHWC activations: no cuDNN layout transposes
                self.pix2pix_model.to(memory_format=torch.channels_last)
        self.pix2pix_model_on_one_gpu = self.pix2pix_model
        net = self.pix2pix_model.net
        if _world() > 1:  # replicas must start identical: rank 0's weights win
            for t in list(self.pix2pix_model.parameters()) + list(self.pix2pix_model.buffers()):
                dist.broadcast(t.data, src=0)
        if opt.use_ema:
            self.netG_ema, self.netCorr_ema = EMA(opt.ema_beta), EMA(opt.ema_beta)
            for ema, key in ((self.netG_ema, "netG"), (self.netCorr_ema, "netCorr")):
                for name, p in net[key].named_parameters():
                    if p.requires_grad:
                        ema.register(name, p.data)
        self.generated = None
        if opt.isTrain:
            self.optimizer_G, self.optimizer_D = self.pix2pix_model.create_optimizers(opt)
            self.old_lr = opt.lr
            if opt.continue_train and opt.which_epoch == "latest":
                ckpt = torch.load(os.path.join(opt.checkpoints_dir, opt.name, "optimizer.pth"), map_location="cpu")
                self.optimizer_G.load_state_dict(ckpt["G"])
                self.optimizer_D.load_state_dict(ckpt["D"])
                self.old_lr = ckpt.get("lr", self.old_lr)  # resume mid-schedule (pix2pix_trainer.py:38-43)
            self._g_params = [p for k in ("netG", "netCorr") for p in net[k].parameters()]
            self._d_params = [p for p in net["netD"].parameters()]
        self.g_losses, self.d_losses, self.out = {}, {}, {}
        self._graph, self._static_in, self._eager_steps, self._side = None, None, 0, None
        self.graph_native_launches = 0
        self.graph_error = None
        self._graph_key_captured = None
        self.pre_sharded = bool(getattr(opt, "pre_sharded", False))
        if opt.isTrain and "COCOS_NATIVE_DGRAD" not in os.environ:
            # K2 backward-data lowers the GPU-busy time but adds launches: it pays off once the iteration is replayed
            # from a graph and costs time on the launch-bound eager step
            from . import ops
            ops.NATIVE_DGRAD = self.graph_capable()

    # ------------------------------------------------------------------ CUDA-graph step (one GPU)
    GRAPH_WARMUP = 3  # eager iterations before the capture (cuDNN autotuning, lazy state, allocator warm-up)

    def graph_capable(self):
        # with more than one rank the gradient all-reduce is captured with the iteration (NCCL only)
        return (self.opt.isTrain and len(self.opt.gpu_ids) > 0 and (_world() == 1 or dist.get_backend() == "nccl")
                and os.environ.get("COCOS_CUDA_GRAPH", "1") == "1" and self.graph_error is None)

    def _eager_step(self, data, alpha=1):
        self.run_generator_one_step(data, alpha)
        self.run_discriminator_one_step(data)

    def _load_static(self, data):
        for k, buf in self._static_in.items():
            buf.copy_(data[k], non_blocking=True)

    def run_step(self, data, alpha=1):
        """One full training iteration (== run_generator_one_step + run_discriminator_one_step, train.py:55-59).
        Every call is exactly one optimiser step of G and of D.  On one GPU (COCOS_CUDA_GRAPH=0 turns it off) the first GRAPH_WARMUP calls run eagerly,
        the next one captures the iteration into a CUDA graph, and from then on a call is: copy the batch into the
        static input buffers (host or device source) + one graph launch.  `alpha`, the learning rates and the batch
        shapes are baked into the graph (update_learning_rate drops it; it is re-captured on the next call)."""
        if not self.graph_capable():
            return self._eager_step(data, alpha)
        key = self._graph_key(alpha)
        if self._graph is not None and key != self._graph_key_captured:
            self._graph = None  # a value the step reads from Python changed: re-capture with it
        if self._graph is None:
            for pg in self.optimizer_G.param_groups + self.optimizer_D.param_groups:
                pg["capturable"] = True  # before the first step: Adam's step counters live on the device
            if self._eager_steps < self.GRAPH_WARMUP:
                # on a side stream: modules that keep a piece of the autograd graph between iterations (spectral
                # norm's cached `weight`) keep the parameters' AccumulateGrad nodes alive, and a node born on the
                # legacy default stream cannot be used from a capturing stream
                self._eager_steps += 1
                if self._side is None:
                    self._side = torch.cuda.Stream()
                self._side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(self._side):
                    self._eager_step(data, alpha)
                torch.cuda.current_stream().wait_stream(self._side)
                return None
            self._capture(data, alpha)
            if self._graph is None:  # capture failed: stay eager, loudly
                return self._eager_step(data, alpha)
        if any(tuple(data[k].shape) != tuple(buf.shape) for k, buf in self._static_in.items()):
            return self._eager_step(data, alpha)  # e.g. the short last batch of an epoch: not the captured shapes
        self._load_static(data)
        self._graph.replay()
        nhwc.clear_pack_cache()  # the replay changed parameters without bumping their version counters

    def free_graph(self):
        """Drop the captured iteration and its private memory pool (it is re-captured on the next run_step)."""
        self._graph = self._static_in = None
        self._graph_key_captured = None
        self.g_losses, self.d_losses, self.out = {}, {}, {}

    def _graph_key(self, alpha):
        """Everything the iteration reads from Python (and therefore bakes into a captured graph): alpha -- only the
        gradient-reversal layer of the domain classifier reads it (correspondence.py:296-300, --weight_domainC > 0), it
        changes every iteration there, so those configs are better left eager -- and the epoch-dependent branch of
        NoVGGCorrespondence.forward (--noise_for_mask after --mask_epoch, correspondence.py:254-258); the learning
        rate is handled by update_learning_rate."""
        opt = self.opt
        return (float(alpha) if opt.weight_domainC > 0 else None, bool(getattr(opt, "noise_for_mask", False)
                                   and getattr(opt, "epoch", 0) > getattr(opt, "mask_epoch", 0)))

    def _capture(self, data, alpha):
        from . import _lib
        self._static_in = {k: torch.empty_like(v, device="cuda") for k, v in data.items() if torch.is_tensor(v)}
        static = dict(data)
        static.update(self._static_in)
        self._load_static(data)
        # The eager iterations ran on the default stream and their autograd graphs (kept alive by the loss / output
        # dicts) pin every parameter's AccumulateGrad node to that stream; a backward captured on the side stream
        # would then have to synchronise with the legacy stream, which invalidates the capture.  Drop them first.
        import gc
        self.g_losses, self.d_losses, self.out = {}, {}, {}
        self.optimizer_G.zero_grad(set_to_none=True)
        self.optimizer_D.zero_grad(set_to_none=True)
        gc.collect()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        nhwc.clear_pack_cache()  # everything the graph reads must be produced inside it (or be immutable)
        l0 = _lib.LAUNCHES
        err = None
        try:
            # thread_local: NCCL's watchdog thread may query events while this thread captures
            with torch.cuda.graph(graph, capture_error_mode="thread_local" if _world() > 1 else "global"):
                self._eager_step(static, alpha)
        except Exception as e:  # noqa: BLE001 -- an op that cannot be captured: report it and keep training eagerly
            err = "%s: %s" % (type(e).__name__, str(e).splitlines()[0] if str(e) else "")
        if _world() > 1:  # all ranks replay or none does
            flag = torch.tensor([0.0 if err is None else 1.0], device="cuda")
            dist.all_reduce(flag)
            if float(flag.item()) > 0 and err is None:
                err = "capture failed on another rank"
        if err is not None:
            self.graph_error = err
            print("cocosnet_b200: CUDA-graph capture of the train step failed (%s); running eagerly" % self.graph_error)
            if os.environ.get("COCOS_GRAPH_TRACE", "0") == "1":
                import traceback
                traceback.print_exc()
            torch.cuda.synchronize()
            self._static_in = None
            if "COCOS_NATIVE_DGRAD" not in os.environ:
                from . import ops
                ops.NATIVE_DGRAD = False  # the eager setting (see __init__)
            return
        self.graph_native_launches = _lib.LAUNCHES - l0
        self._graph = graph
        nhwc.clear_pack_cache()  # buffers packed during the capture live in the graph's pool: not for eager use
        self._graph_key_captured = self._graph_key(alpha)

    def _shard(self, data):
        """This rank's slice of a global batch; `pre_sharded` = the caller already hands over rank-local batches
        (a per-rank data loader, bench.py's weak-scaling batches)."""
        return data if self.pre_sharded else shard_batch(data)

    def run_generator_one_step(self, data, alpha=1):
        self.optimizer_G.zero_grad(set_to_none=True)
        # The G step only needs the gradient THROUGH the discriminator, not its weight gradients (the reference
        # computes and then discards them: optimizer_D.zero_grad() runs before they are ever used).
        for p in self._d_params:
            p.requires_grad_(False)
        # more than one rank (NCCL): the generator's gradients are complete as soon as the backward leaves netG -- the
        # hook the model places on netCorr's output fires there -- so their all-reduce (62 % of the bytes) runs on
        # NCCL's stream underneath netCorr's backward; the rest follows after the backward
        overlap = _world() > 1 and dist.get_backend() == "nccl" and "warp" in self.opt.CBN_intype \
            and os.environ.get("COCOS_OVERLAP_ALLREDUCE", "1") == "1"
        pending = []
        if overlap:
            netg = [p for p in self.pix2pix_model.net["netG"].parameters() if p.requires_grad]

            def early():
                # every netG parameter receives exactly one gradient per step and .grad was None before: all present
                # == all final (otherwise nothing is started here and the whole set is reduced after the backward)
                if all(p.grad is not None for p in netg):
                    pending.append(allreduce_grads(netg, async_op=True))
            self.pix2pix_model.after_netG_backward = early
        try:
            g_losses, out = self.pix2pix_model(self._shard(data), mode="generator", alpha=alpha)
            g_loss = sum(g_losses.values()).mean()
            g_loss.backward()
        finally:
            self.pix2pix_model.after_netG_backward = None
            for p in self._d_params:
                p.requires_grad_(True)
        self.g_losses, self.out = g_losses, out
        if overlap and pending:
            allreduce_grads([p for p in self.pix2pix_model.net["netCorr"].parameters()])
        else:
            allreduce_grads(self._g_params)
            pending = []

        for h in pending:  # netG's early all-reduce
            if h is not None:
                h.wait()
        self.optimizer_G.step()
        if self.opt.use_ema:
            self.netG_ema(self.pix2pix_model.net["netG"])
            self.netCorr_ema(self.pix2pix_model.net["netCorr"])

    def run_discriminator_one_step(self, data):
        self.optimizer_D.zero_grad(set_to_none=True)
        GforD = {k: self.out.get(k) for k in ("fake_image", "adaptive_feature_seg", "adaptive_feature_img")}
        d_losses = self.pix2pix_model(self._shard(data), mode="discriminator", GforD=GforD)
        d_loss = sum(d_losses.values()).mean()
        d_loss.backward()
        allreduce_grads(self._d_params)
        self.optimizer_D.step()
        self.d_losses = d_losses

    def get_latest_losses(self):
        return {**self.g_losses, **self.d_losses}

    def get_latest_generated(self):
        return self.out["fake_image"]

    def save(self, epoch):
        if _rank() != 0:
            return
        model = self.pix2pix_model
        model.save(epoch)
        if self.opt.use_ema:
            for ema, key, label in ((self.netG_ema, "netG", "G_ema"), (self.netCorr_ema, "netCorr", "netCorr_ema")):
                ema.assign(model.net[key])
                util.save_network(model.net[key], label, epoch, self.opt)
                ema.resume(model.net[key])
        if epoch == "latest":
            torch.save({"G": self.optimizer_G.state_dict(), "D": self.optimizer_D.state_dict(), "lr": self.old_lr},
                       os.path.join(self.opt.checkpoints_dir, self.opt.name, "optimizer.pth"))

    def update_learning_rate(self, epoch):
        new_lr = self.old_lr - self.opt.lr / self.opt.niter_decay if epoch > self.opt.niter else self.old_lr
        if new_lr != self.old_lr:
            g_lr, d_lr = (new_lr, new_lr) if self.opt.no_TTUR else (new_lr / 2, new_lr * 2)
            for pg in self.optimizer_D.param_groups:
                pg["lr"] = d_lr
            for pg in self.optimizer_G.param_groups:
                pg["lr"] = g_lr
            print("update learning rate: %f -> %f" % (self.old_lr, new_lr))
            self.old_lr = new_lr
            self._graph = None  # the learning rate is a launch constant of the captured fused-Adam kernels
