"""Data-parallel update step for the SpeechT5 hot path (host side).

Mirrors what fairseq does around the model for one update -- fairseq/trainer.py:675-952 (zero_grad -> per-micro-batch
task.train_step -> all_reduce_grads -> multiply_grads(world / sample_size) -> clip_grad_norm -> optimizer.step) with
LegacyDistributedDataParallel semantics for the gradient exchange (legacy_distributed_data_parallel.py:76-165: grads
/= world, all-reduce(sum), parameters without a gradient contribute zeros) -- re-designed for H100:

  * parameters, gradients, Adam moments live in single flat fp32 buffers plus a flat bf16 shadow; fused operand groups
    (q|k|v weights, k|v, feat_out|prob_out, and their biases) are laid out adjacently so the GEMMs read them in place;
  * the flat buffers are ordered by STAGE (one per encoder / decoder layer, forward order): the GEMM weights of a stage
    form one contiguous, world-divisible range, everything small (biases, norms, embeddings, conv filters) sits in a
    replicated tail;
  * gradient exchange (world > 1), `exchange="shard"` (default in bf16 mode): when autograd delivers the gradient of a
    stage's INPUT, every weight gradient of that stage is final -- its range is REDUCE-SCATTERED (NCCL over NVLink) on a
    side stream while the earlier stages are still in backward; each rank then owns 1/world of every stage: squared
    norm of its shards (+ one 4-byte all-reduce), clip + Adam + bf16-shadow refresh on the shards only (the optimizer
    pass shrinks by the world size), and the updated bf16 shards are ALL-GATHERED back into every rank's flat shadow,
    which is the only thing the GEMMs read. fp32 masters of the sharded ranges are valid on their owner only until
    `consolidate()` (state_dict / evaluation in parity mode call it). `exchange="allreduce"`: the same per-stage
    overlap with plain fp32 all-reduce and a replicated optimizer (parity mode, CPU / gloo);
  * clip + Adam + bf16-shadow refresh is one kernel launch per contiguous range (st5_adam_step), lr / step in device
    memory; a non-finite gradient norm skips the update on the device (overflow counter, `check_overflow`);
  * the whole update (zero, forward, backward, exchange, norm, Adam, gather) is captured into a CUDA graph per input
    shape signature and replayed; graphs are kept in an LRU cache, a cache miss captures WITHOUT running warm-up updates
    (capture executes nothing, so ranks never disagree on the number of collectives), optional padding of the time axes
    to bucket multiples keeps the number of signatures small;
  * LayerDrop (encoder.py:251-257, decoder LayerDropModuleList) under capture: the host draws the layer subset like the
    reference (numpy RNG for the encoder, torch RNG for the decoder) into a device mask; a dropped layer's output is
    replaced by its input, so its parameters get exactly zero gradient (eager mode really skips the layer).
"""
import collections
import os

import numpy as np
import torch
import torch.distributed as dist

from . import kernels as K
from .models.modules.transformer import MultiheadAttention
from .ops import RT


class GradBucketer:
    """Mean-reduces a flat gradient buffer across ranks in fixed-size buckets. Device agnostic (NCCL or gloo)."""

    def __init__(self, flat_grads, bucket_elems=32 * 1024 * 1024, group=None):
        self.flat = flat_grads
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        n = flat_grads.numel()
        self.bounds = [(s, min(n, s + bucket_elems)) for s in range(0, n, bucket_elems)]

    def all_reduce_mean(self):
        if self.world == 1:
            return
        for s, e in self.bounds:
            chunk = self.flat[s:e]
            chunk.div_(self.world)  # legacy_ddp.py:110 (div before the sum keeps fp16/bf16 ranges safe)
            dist.all_reduce(chunk, op=dist.ReduceOp.SUM, group=self.group)

    def all_reduce_sum(self, lo=0, hi=None):
        """Sum (not mean) of flat[lo:hi] over the ranks, bucket by bucket; the caller folds 1/world into the gradient
        multiplier it applies anyway (fp32 buffer: no range concern, one elementwise pass over the buffer less)."""
        if self.world == 1:
            return
        hi = self.flat.numel() if hi is None else hi
        step = self.bounds[0][1] - self.bounds[0][0] if self.bounds else hi
        for s in range(lo, hi, max(1, step)):
            dist.all_reduce(self.flat[s:min(hi, s + step)], op=dist.ReduceOp.SUM, group=self.group)


def _fused_groups(model):
    """Parameter groups that must be adjacent in the flat buffers (read as one fused GEMM operand)."""
    groups = []
    for m in model.modules():
        if isinstance(m, MultiheadAttention):
            if m.self_attention:
                groups.append([m.q_proj.weight, m.k_proj.weight, m.v_proj.weight])
                groups.append([m.q_proj.bias, m.k_proj.bias, m.v_proj.bias])
            else:
                groups.append([m.k_proj.weight, m.v_proj.weight])
                groups.append([m.k_proj.bias, m.v_proj.bias])
    post = getattr(model, "speech_decoder_postnet", None)
    if post is not None:
        groups.append([post.feat_out.weight, post.prob_out.weight])
        groups.append([post.feat_out.bias, post.prob_out.bias])
    return [g for g in groups if all(p is not None for p in g)]


def stage_of(name, group=1):
    """Stage key of a parameter name: ("enc", g) / ("dec", g) for the transformer layers (g = layer // group: `group`
    consecutive layers form one exchange stage), None for everything else."""
    for prefix, tag in (("encoder.layers.", "enc"), ("decoder.layers.", "dec")):
        if name.startswith(prefix):
            return (tag, int(name[len(prefix):].split(".", 1)[0]) // max(1, group))
    return None


class FlatParams:
    """Flat fp32 master / gradient / moment buffers + flat bf16 shadow, `nn.Parameter`s re-pointed to views.

    Layout: [stage 0 GEMM weights | stage 1 ... | stage S-1 | replicated tail]. A stage range is padded to a multiple
    of 8 * world elements (16-byte bf16 alignment of every shard). `stages` maps stage key -> (lo, hi)."""

    def __init__(self, model, world=1, rank=0, stage_group=1):
        params = [p for p in model.parameters()]
        self.stage_group = max(1, int(stage_group))
        dev = params[0].device
        self.world, self.rank = world, rank
        groups = _fused_groups(model)
        in_group = {id(p) for g in groups for p in g}
        gmap = {id(g[0]): g for g in groups}
        names = {id(p): n for n, p in model.named_parameters()}
        units, seen = [], set()  # a unit = a fused group or a single parameter, in parameters() order
        for p in params:
            if id(p) in seen:
                continue
            if id(p) in gmap:
                units.append(gmap[id(p)])
                seen.update(id(q) for q in gmap[id(p)])
            elif id(p) not in in_group:
                units.append([p])
                seen.add(id(p))
        for g in groups:  # groups whose first member was not met first in parameters() order
            if id(g[0]) not in seen:
                units.append(g)
                seen.update(id(q) for q in g)

        def key(u):  # stage of a unit; only 2-D GEMM weights (static flat shadows) are placed in stage ranges
            return stage_of(names.get(id(u[0]), ""), self.stage_group) if u[0].dim() == 2 else None
        order_keys = sorted({key(u) for u in units if key(u) is not None}, key=lambda k: (k[0] != "enc", k[1]))
        offsets, off = {}, 0
        self.stages = collections.OrderedDict()
        align = 8 * max(1, world)
        for sk in order_keys:
            lo = off
            for u in units:
                if key(u) == sk:
                    off = (off + 7) // 8 * 8
                    for p in u:
                        offsets[id(p)] = off
                        off += p.numel()
            off = lo + (off - lo + align - 1) // align * align
            self.stages[sk] = (lo, off)
        self.tail = off
        for u in units:
            if key(u) is None:
                off = (off + 7) // 8 * 8  # 16-byte alignment of every bf16 operand (TMA)
                for p in u:
                    offsets[id(p)] = off
                    off += p.numel()
        self.numel = (off + 7) // 8 * 8
        self.flat = torch.zeros(self.numel, dtype=torch.float32, device=dev)
        self.grads = torch.zeros_like(self.flat)
        self.exp_avg = torch.zeros_like(self.flat)
        self.exp_avg_sq = torch.zeros_like(self.flat)
        self.shadow = torch.zeros(self.numel, dtype=torch.bfloat16, device=dev)
        self.offsets = offsets
        with torch.no_grad():
            for p in params:
                o, n = offsets[id(p)], p.numel()
                self.flat[o:o + n].copy_(p.detach().reshape(-1))
                p.data = self.flat[o:o + n].view(p.shape)
                p.grad = self.grads[o:o + n].view(p.shape)
        self.refresh_shadow()
        # static shadows / fused biases for ops.linear
        RT.clear_static()
        for p in params:
            if p.dim() == 2:
                o = offsets[id(p)]
                RT.register_static(("lin", id(p)), self.shadow[o:o + p.numel()].view(p.shape))
                RT.register_static_grad(("lin", id(p)), self.grads[o:o + p.numel()].view(p.shape))
            elif p.dim() == 1:
                o = offsets[id(p)]
                RT.register_static_grad(("bias", id(p)), self.grads[o:o + p.numel()])
        for g in groups:
            o = offsets[id(g[0])]
            n = sum(p.numel() for p in g)
            if g[0].dim() == 2:
                RT.register_static(("lin",) + tuple(id(p) for p in g), self.shadow[o:o + n].view(-1, g[0].shape[1]))
                RT.register_static_grad(("lin",) + tuple(id(p) for p in g), self.grads[o:o + n].view(-1, g[0].shape[1]))
            else:
                RT.register_static(("bias",) + tuple(id(p) for p in g), self.flat[o:o + n])
                RT.register_static_grad(("bias",) + tuple(id(p) for p in g), self.grads[o:o + n])
        RT.register_static_refresh(self.refresh_shadow)
        self.params = params

    def shard(self, sk, rank=None):
        """(lo, hi) of `rank`'s shard of stage `sk`."""
        lo, hi = self.stages[sk]
        c = (hi - lo) // self.world
        r = self.rank if rank is None else rank
        return lo + r * c, lo + (r + 1) * c

    def refresh_shadow(self):
        K.cast_bf16(self.flat.view(1, -1), self.shadow.view(1, -1))
        RT.invalidate_shadows()


class B200Trainer:
    """One process per GPU. `train_step(samples)` == fairseq Trainer.train_step for the speecht5 task."""

    def __init__(self, model, criterion, task, lr=1e-4, betas=(0.9, 0.98), eps=1e-8, weight_decay=0.0, clip_norm=25.0,
                 process_group=None, use_cuda_graph=True, bucket_mb=128, exchange=None, graph_cache=8,
                 shape_buckets=None, stage_group=3):
        self.model, self.criterion, self.task = model, criterion, task
        self.lr, self.betas, self.eps, self.weight_decay, self.clip_norm = lr, betas, eps, weight_decay, clip_norm
        self.device = next(model.parameters()).device
        self.criterion.to(self.device)  # criterion buffers (BCE pos_weight) must live on the device for capture
        # the guided-attention loss reads the first n heads of every cross-attention map (text_to_speech_loss.py:210-212):
        # the attention backward need not read the (zero) gradient of the other heads
        t2s = getattr(criterion, "text_to_speech_loss", None)
        RT.probs_grad_heads = (int(getattr(t2s, "num_heads_applied_guided_attn", 0))
                               if (t2s is not None and getattr(t2s, "use_guided_attn_loss", False)) else 0)
        # ... and inside an update the criterion is the ONLY reader of the returned maps: the forward need not write the
        # other heads' probabilities at all (77 MB of fp32 per decoder layer at the benched shape). Scoped to train_step.
        self._probs_read_heads = RT.probs_grad_heads
        self._prefetched, self._staging, self._staging_read = None, {}, None
        self._gate_thresholds = None
        self._frame_pm_cache = {}
        self._wgrad_side = False  # (set below once the world size is known)
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank(process_group) if self.world > 1 else 0
        # weight-gradient GEMMs on a second stream (ops.wgrad_mm): +1.1 % at N = 1; the stage collectives wait for it
        self._wgrad_side = os.environ.get("ST5_WGRAD_SIDE", "1") != "0" and self.device.type == "cuda"
        RT.wgrad_stream = None
        self._wgrad_stream = None
        if exchange is None:
            exchange = os.environ.get("ST5_EXCHANGE") or ("shard" if RT.dtype == torch.bfloat16 else "allreduce")
        assert exchange in ("shard", "allreduce")
        if RT.dtype == torch.float32 and exchange == "shard" and self.world > 1:
            raise ValueError("parity mode reads the fp32 masters in every GEMM: use exchange='allreduce'")
        self.exchange = exchange if self.world > 1 else "none"
        # layers per exchange stage: fewer, larger collectives (each NCCL launch has to squeeze its CTAs in between
        # persistent 132-CTA GEMM grids) against later overlap; ST5_STAGE_GROUP overrides
        self.stage_group = int(os.environ.get("ST5_STAGE_GROUP", stage_group))
        self.fp = FlatParams(model, self.world if self.exchange == "shard" else 1, self.rank, self.stage_group)
        self.bucketer = GradBucketer(self.fp.grads, bucket_elems=bucket_mb * 1024 * 1024 // 4, group=process_group)
        # overlap of the exchange with backward: model code calls RT.stage(key, x) at the entry of every stage
        self._overlap = self.world > 1 and os.environ.get("ST5_OVERLAP_AR", "1") != "0"
        self._side = torch.cuda.Stream(device=self.device) if (self._overlap and self.device.type == "cuda") else None
        self._done, self._last_micro = set(), False
        self.overlapped_stages = 0  # stages whose exchange was launched from the backward hook (all-time counter)
        self._sharded_dirty = False  # fp32 masters / moments of foreign shards are stale (exchange == "shard")
        RT.stage_callback = self._on_stage if self.world > 1 else None
        self.num_updates = 0
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.lr_dev = torch.full((1,), lr, dtype=torch.float32, device=self.device)
        self.gnorm_sq = torch.zeros(1, dtype=torch.float32, device=self.device)
        self._gn_tail = torch.zeros(1, dtype=torch.float32, device=self.device)
        self.overflow_dev = torch.zeros(1, dtype=torch.int64, device=self.device)  # updates skipped: non-finite norm
        self.use_cuda_graph = use_cuda_graph and self.device.type == "cuda"
        self.graph_cache_size = graph_cache
        self.shape_buckets = shape_buckets  # e.g. {"text": 32, "frames": 64}: pad the time axes to these multiples
        self._graphs = collections.OrderedDict()  # signature -> (graph, static samples, static out)
        self._warmed = False
        self.graph_hits = self.graph_misses = 0
        # LayerDrop: one keep flag per encoder / decoder layer, drawn on the host per update
        self._n_enc = len(getattr(model.encoder, "layers", []))
        self._n_dec = len(getattr(model.decoder, "layers", []))
        self.layer_keep = torch.ones(self._n_enc + self._n_dec, dtype=torch.float32, device=self.device)
        self._keep_host = torch.ones(self._n_enc + self._n_dec, dtype=torch.float32)
        if self.device.type == "cuda":
            self._keep_host = self._keep_host.pin_memory()
            RT.enable_device_seed(self.device)

    # ------------------------------------------------------------------ exchange
    def _collective(self, fn):
        """Run a collective on the side stream (ordered after everything issued so far on the current stream)."""
        if self._side is None:
            fn()
            return
        self._side.wait_stream(torch.cuda.current_stream())
        if RT.wgrad_stream is not None and RT._side_keep:  # the weight gradients this collective moves were written there
            self._side.wait_stream(RT.wgrad_stream)
        with torch.cuda.stream(self._side):
            fn()

    def _reduce_stage(self, sk):
        lo, hi = self.fp.stages[sk]
        g = self.fp.grads[lo:hi]
        if self.exchange == "shard":
            slo, shi = self.fp.shard(sk)
            own = self.fp.grads[slo:shi]
            try:
                dist.reduce_scatter_tensor(own, g, op=dist.ReduceOp.SUM, group=self.group)
            except (RuntimeError, NotImplementedError):  # gloo has no reduce-scatter: same result from an all-reduce
                dist.all_reduce(g, op=dist.ReduceOp.SUM, group=self.group)
        else:
            dist.all_reduce(g, op=dist.ReduceOp.SUM, group=self.group)

    def _on_stage(self, sk, x):
        """Called by the model at the entry of stage `sk` (forward). In backward, the gradient of this tensor arrives
        after every parameter gradient of the stage has been written: launch the stage's exchange there."""
        tag, idx = sk
        if idx % self.stage_group != 0:  # the gradient of a GROUP's first layer input is the last one of the group
            return x
        sk = (tag, idx // self.stage_group)
        if sk in self.fp.stages and self._overlap and torch.is_grad_enabled() and x.requires_grad:
            def hook(grad, sk=sk):
                if self._last_micro and sk not in self._done:
                    self._done.add(sk)
                    self.overlapped_stages += 1
                    self._collective(lambda: self._reduce_stage(sk))
                return None
            x.register_hook(hook)
        return x

    def _finish_exchange(self):
        """Stages whose hook did not fire (frozen, dropped, no overlap) + the replicated tail; join the side stream."""
        for sk in reversed(self.fp.stages):
            if sk not in self._done:
                self._done.add(sk)
                self._collective(lambda sk=sk: self._reduce_stage(sk))
        if self.fp.tail < self.fp.numel:
            self._collective(lambda: self.bucketer.all_reduce_sum(self.fp.tail, self.fp.numel))
        if self._side is not None:
            torch.cuda.current_stream().wait_stream(self._side)

    def _owned_ranges(self):
        """Contiguous ranges this rank runs the optimizer on."""
        if self.exchange != "shard":
            return [(0, self.fp.numel)]
        return [self.fp.shard(sk) for sk in self.fp.stages] + [(self.fp.tail, self.fp.numel)]

    # ------------------------------------------------------------------ the update, as a sequence of device work
    def _update(self, samples):
        if self._wgrad_side and self._wgrad_stream is None:
            self._wgrad_stream = torch.cuda.Stream(device=self.device)
        self.fp.grads.zero_()
        losses, stats = [], []
        self._done = set()
        # the side stream is visible to the ops only while this update's backward passes run: a backward issued outside
        # the trainer (tests, user code) must not leave work on a stream nobody joins
        RT.wgrad_stream = self._wgrad_stream
        try:
            for k, sample in enumerate(samples):  # --update-freq micro-batches
                self._last_micro = k == len(samples) - 1
                loss, sample_size, logging_output = self.task.train_step(sample, self.model, self.criterion, None,
                                                                         self.num_updates)
                losses.append(loss if torch.is_tensor(loss) else torch.tensor(loss, device=self.device))
                stats.append(logging_output.get(sample["task_name"], logging_output).get("_stats"))
            self._last_micro = False
            RT.side_join()
        finally:
            RT.wgrad_stream = None
        if self.world > 1:
            self._finish_exchange()
        # legacy_ddp.py:110 divides by world before the sum; trainer.py:796 multiply_grads(world / sample_size) with
        # sample_size = world * n_micro (every micro-batch on every rank reports 1). Net factor on the summed gradient:
        grad_mul = self._grad_mul = 1.0 / float(self.world * len(samples))
        self.gnorm_sq.zero_()
        if self.exchange == "shard":
            for lo, hi in self._owned_ranges()[:-1]:
                K.sumsq(self.fp.grads[lo:hi], self.gnorm_sq)
            self._gn_tail.zero_()
            K.sumsq(self.fp.grads[self.fp.tail:], self._gn_tail)  # identical on every rank: count it once
            self.gnorm_sq += self._gn_tail / self.world
            dist.all_reduce(self.gnorm_sq, op=dist.ReduceOp.SUM, group=self.group)
        else:
            K.sumsq(self.fp.grads, self.gnorm_sq)
        finite = torch.isfinite(self.gnorm_sq)
        self.step_dev += finite  # a skipped update does not advance Adam's bias correction
        self.overflow_dev += ~finite
        for lo, hi in self._owned_ranges():
            if hi > lo:
                K.adam_step(self.fp.flat[lo:hi], self.fp.grads[lo:hi], self.fp.exp_avg[lo:hi], self.fp.exp_avg_sq[lo:hi],
                            self.fp.shadow[lo:hi], self.lr, self.betas[0], self.betas[1], self.eps, self.weight_decay, 1,
                            self.gnorm_sq, self.clip_norm, grad_mul, lr_dev=self.lr_dev, step_dev=self.step_dev)
        if self.exchange == "shard":
            self._gather(self.fp.shadow)  # every rank's updated bf16 shards -> every rank's flat shadow
            self._sharded_dirty = True
        RT.advance_seed()
        return torch.stack(losses), (torch.stack(stats) if stats[0] is not None else None)

    def _gather(self, buf):
        """Every rank's shard of every stage -> every rank's full stage range. On NCCL the per-stage all-gathers are
        issued as ONE coalesced group (a single launch instead of one per layer: they all sit, exposed, at the end of
        the update)."""
        stages = list(self.fp.stages)
        if self.device.type == "cuda" and len(stages) > 1 and os.environ.get("ST5_COALESCE", "1") != "0":
            try:
                from torch.distributed.distributed_c10d import _coalescing_manager
                with _coalescing_manager(group=self.group, device=self.device, async_ops=False):
                    for sk in stages:
                        lo, hi = self.fp.stages[sk]
                        slo, shi = self.fp.shard(sk)
                        dist.all_gather_into_tensor(buf[lo:hi], buf[slo:shi], group=self.group)
                return
            except (ImportError, RuntimeError, NotImplementedError):
                pass
        for sk in stages:
            lo, hi = self.fp.stages[sk]
            slo, shi = self.fp.shard(sk)
            try:
                dist.all_gather_into_tensor(buf[lo:hi], buf[slo:shi], group=self.group)
            except (RuntimeError, NotImplementedError):
                parts = [torch.empty_like(buf[slo:shi]) for _ in range(self.world)]
                dist.all_gather(parts, buf[slo:shi].clone(), group=self.group)
                buf[lo:hi].copy_(torch.cat(parts))

    def consolidate(self):
        """exchange == "shard": bring the fp32 masters and Adam moments of the foreign shards up to date on this rank
        (checkpointing, evaluation in parity mode, leaving sharded training). Collective: every rank must call it."""
        if self.exchange == "shard" and self._sharded_dirty:
            for buf in (self.fp.flat, self.fp.exp_avg, self.fp.exp_avg_sq):
                self._gather(buf)
            self._sharded_dirty = False

    def grad_norm(self):
        """Gradient norm of the last update as the reference computes it (after multiply_grads, before clipping)."""
        return float(self.gnorm_sq.sqrt().item()) * getattr(self, "_grad_mul", 1.0)

    def check_overflow(self):
        """fairseq/trainer.py:845-858 raises FloatingPointError when the gradient norm is NaN / Inf; the device skips
        such an update and counts it -- call this wherever a host sync is acceptable (log interval)."""
        n = int(self.overflow_dev.item())
        if n > 0:
            self.overflow_dev.zero_()
            raise FloatingPointError(f"gradients are NaN/Inf in {n} update(s); those updates were skipped")

    # ------------------------------------------------------------------ optimizer state (fairseq/optim/adam.py layout)
    def state_dict(self):
        """Optimizer state in fairseq's checkpoint layout (`last_optimizer_state`: torch.optim-style {"state": {i: {step,
        exp_avg, exp_avg_sq}}, "param_groups": [...]}, parameters indexed in model.parameters() order) + counters."""
        self.consolidate()
        step = int(self.step_dev.item())
        state = {}
        for i, p in enumerate(self.fp.params):
            o, n = self.fp.offsets[id(p)], p.numel()
            state[i] = {"step": step, "exp_avg": self.fp.exp_avg[o:o + n].view(p.shape).clone(),
                        "exp_avg_sq": self.fp.exp_avg_sq[o:o + n].view(p.shape).clone()}
        group = {"lr": self.lr, "betas": tuple(self.betas), "eps": self.eps, "weight_decay": self.weight_decay,
                 "amsgrad": False, "params": list(range(len(self.fp.params)))}
        return {"state": state, "param_groups": [group], "num_updates": self.num_updates,
                "dropout_seed": int(RT._seed_t.item()) if RT._seed_t is not None else RT._seed}

    def load_state_dict(self, sd):
        with torch.no_grad():
            for i, p in enumerate(self.fp.params):
                st = sd["state"].get(i)
                if st is None:
                    continue
                o, n = self.fp.offsets[id(p)], p.numel()
                self.fp.exp_avg[o:o + n].copy_(st["exp_avg"].reshape(-1))
                self.fp.exp_avg_sq[o:o + n].copy_(st["exp_avg_sq"].reshape(-1))
                self.step_dev.fill_(int(st["step"]))
        g = sd["param_groups"][0]
        self.lr, self.betas, self.eps, self.weight_decay = g["lr"], tuple(g["betas"]), g["eps"], g["weight_decay"]
        self.lr_dev.fill_(self.lr)
        self.num_updates = sd.get("num_updates", self.num_updates)
        if "dropout_seed" in sd:
            RT.manual_seed(sd["dropout_seed"])
        self._graphs.clear()  # captured graphs bake the betas / eps scalars

    # ------------------------------------------------------------------ LayerDrop
    def _draw_layerdrop(self):
        """Host draw of this update's layer subset, in the reference's RNG streams and order: one numpy uniform per
        encoder layer (encoder.py:252), one torch uniform per decoder layer (fairseq LayerDropModuleList)."""
        enc_p = float(getattr(self.model.encoder, "encoder_layerdrop", 0.0) or 0.0)
        dec_p = float(getattr(self.model.decoder, "decoder_layerdrop", 0.0) or 0.0)
        if not self.model.training or (enc_p <= 0 and dec_p <= 0):
            return False
        keep = self._keep_host
        unb = getattr(self.model.encoder, "unb_enc_layer", -1)
        for i in range(self._n_enc):
            keep[i] = 1.0 if (np.random.random() > enc_p or i == unb) else 0.0
        for i in range(self._n_dec):
            keep[self._n_enc + i] = 1.0 if (dec_p <= 0 or torch.empty(1).uniform_().item() > dec_p) else 0.0
        self.layer_keep.copy_(keep, non_blocking=True)
        return True

    def _with_host_draws(self, sample):
        """Speech input: the HuBERT-style time / channel masks are drawn by numpy on the host in the reference
        (speech_encoder_prenet.py:234-272, inside forward). A captured step cannot do that, so the trainer draws them
        here -- same stream, same order -- and hands them to forward() as explicit inputs."""
        prenet = getattr(self.model, "speech_encoder_prenet", None)
        ni = sample.get("net_input", {})
        if (sample.get("task_name") != "s2t" or prenet is None or not self.model.training or "mask_indices" in ni
                or (prenet.mask_prob <= 0 and getattr(prenet, "mask_channel_prob", 0.0) <= 0)):
            return sample
        from .data import draw_hubert_masks
        from .frontend import downsample_padding_mask
        B, n = ni["source"].shape
        T = int(prenet.feature_extractor.get_out_seq_lens_tensor(torch.tensor([n]))[0])
        pm = ni.get("padding_mask")
        frame_pm = None
        if pm is not None:
            # the frame-level padding mask of a batch is a function of its sample-level mask only: remember it per mask
            # tensor (object + version), so that a batch that already lives on the device does not cost a device->host
            # read -- and a drained pipeline -- every time it is stepped on
            key = (id(pm), pm._version, tuple(pm.shape))
            hit = self._frame_pm_cache.get(key)
            if hit is not None and hit[0]() is pm:
                frame_pm = hit[1]
            else:
                import weakref
                frame_pm = downsample_padding_mask(pm.cpu(), T)
                if len(self._frame_pm_cache) >= 64:
                    self._frame_pm_cache.pop(next(iter(self._frame_pm_cache)))
                self._frame_pm_cache[key] = (weakref.ref(pm), frame_pm)
        mi, mc = draw_hubert_masks(prenet, B, T, frame_pm)
        extra = {}
        if mi is not None:
            extra["mask_indices"] = mi.pin_memory() if self.device.type == "cuda" else mi
        if mc is not None:
            extra["mask_channel_indices"] = mc.pin_memory() if self.device.type == "cuda" else mc
        out = dict(sample)
        out["net_input"] = dict(ni, **extra)
        return out

    # ------------------------------------------------------------------ public step
    def _signature(self, samples):
        shapes = tuple(tuple((k, tuple(v.shape)) for k, v in _flatten(s).items()) + (s.get("task_name"),) for s in samples)
        if self._gate_thresholds is None:  # (walking ~500 modules every update cost more host time than the replay call)
            self._gate_thresholds = tuple(
                [getattr(m, "freeze_encoder_updates", 0) for m in self.model.modules() if hasattr(m, "freeze_encoder_updates")]
                + [getattr(m, "freeze_decoder_updates", 0) for m in self.model.modules() if hasattr(m, "freeze_decoder_updates")])
        gates = tuple(t <= self.num_updates for t in self._gate_thresholds)
        return shapes, gates, self.model.training

    def train_step(self, samples, lr=None):
        """samples: list of micro-batch dicts (tensors on host -- pinned for async copies -- or on the device).
        Returns (losses [n_micro] device tensor, stats [n_micro, k] device tensor or None)."""
        RT.probs_read_heads = self._probs_read_heads
        try:
            return self._train_step(samples, lr)
        finally:
            RT.probs_read_heads = 0

    def _train_step(self, samples, lr=None):
        if lr is not None:
            self.lr = lr
            self.lr_dev.fill_(lr)
        for c in (getattr(self.criterion, "text_to_speech_loss", None), getattr(self.criterion, "speech_to_text_loss", None)):
            if c is not None:
                c.defer_logging = True
        pre = self._prefetched
        self._prefetched = None
        staged = None
        if pre is not None and len(pre[0]) == len(samples) and all(a is b for a, b in zip(pre[0], samples)):
            _, samples, staged, ready = pre  # (prepared exactly as below at prefetch time; copies are in flight)
        else:
            if self.shape_buckets:
                samples = [pad_to_buckets(s, self.shape_buckets) for s in samples]
            samples = [self._with_host_draws(s) for s in samples]
        layerdrop = self._draw_layerdrop()
        # the pre-training criteria gather the MASKED frames (a different count every draw) and read their statistics
        # back inside forward (speech_pretrain_criterion.py:101-189): not capturable -- those updates run eagerly
        eager = not self.use_cuda_graph or any(s.get("task_name") in ("speech_pretrain", "text_pretrain") for s in samples)
        if eager:
            RT.layer_keep = None  # eager: the host decides, dropped layers are really skipped
            RT.layer_keep_host = self._keep_host if layerdrop else None
            dev_samples = [_to_device(s, self.device) for s in samples]
            out = self._update(dev_samples)
            RT.layer_keep_host = None
            self.num_updates += 1
            return out
        RT.layer_keep = self.layer_keep if layerdrop else None
        RT.layer_keep_host = None
        sig = self._signature(samples) + (layerdrop,)
        ent = self._graphs.get(sig)
        if ent is None:
            self.graph_misses += 1
            ent = self._capture(samples, sig)
        else:
            self.graph_hits += 1
            self._graphs.move_to_end(sig)
        graph, static_samples, static_out, static_flat = ent
        if staged is not None:  # the host->device copies ran under the previous update: device->device into the graph's inputs
            torch.cuda.current_stream().wait_event(ready)
            staged_views, staged_flat = staged
            if staged_flat.numel() == static_flat.numel():
                static_flat.copy_(staged_flat, non_blocking=True)  # both sets are views of one byte buffer: ONE copy
            else:
                for st, s in zip(static_samples, staged_views):
                    _copy_into(st, s)
            self._staging_read = torch.cuda.Event()
            self._staging_read.record()
        else:
            for st, s in zip(static_samples, samples):
                _copy_into(st, s)
        graph.replay()
        RT.layer_keep = None
        self.num_updates += 1
        return static_out

    def prefetch(self, samples):
        """Input pipeline: start the host->device copies of the NEXT train_step's micro-batches (pinned host tensors) on a
        copy stream, so that they run under the update that is executing now; the next train_step called with the same
        sample objects only moves them device->device into its graph's input buffers. Staging buffers are kept per
        shape signature. A train_step with other samples simply ignores what was prefetched."""
        if not self.use_cuda_graph or self.device.type != "cuda":
            return
        orig = list(samples)
        if self.shape_buckets:
            samples = [pad_to_buckets(s, self.shape_buckets) for s in samples]
        samples = [self._with_host_draws(s) for s in samples]
        shapes = self._signature(samples)[0]
        staging = self._staging.get(shapes)
        if getattr(self, "_h2d_stream", None) is None:
            self._h2d_stream = torch.cuda.Stream(device=self.device)
        with torch.cuda.stream(self._h2d_stream):
            if staging is None:
                if len(self._staging) >= 8:
                    self._staging.pop(next(iter(self._staging)))
                staging = self._staging[shapes] = _to_device_packed(samples, self.device)
            else:
                # the last reader of these buffers: the device->device copies train_step issued BEFORE its graph replay
                # (waiting for the main stream itself would put this copy behind the update it is meant to hide under)
                if self._staging_read is not None:
                    self._h2d_stream.wait_event(self._staging_read)
                for st, s in zip(staging[0], samples):
                    _copy_into(st, s)
            ready = torch.cuda.Event()
            ready.record(self._h2d_stream)
        self._prefetched = (orig, samples, staging, ready)

    def _capture_stream(self):
        if getattr(self, "_cap_stream", None) is None:
            self._cap_stream = torch.cuda.Stream(device=self.device)
        return self._cap_stream

    def _capture(self, samples, sig):
        static_samples, static_flat = _to_device_packed(samples, self.device)
        if not self._warmed:
            # ONE eager update outside capture, first capture only (lazy inits: NCCL communicator, allocator pools,
            # module caches); every rank reaches it at its first step, so the collectives it issues pair up. It is a real
            # update on the first batch; state is restored afterwards so capture leaves the training trajectory alone.
            state = (self.fp.flat, self.fp.exp_avg, self.fp.exp_avg_sq, self.fp.shadow, self.step_dev, self.overflow_dev)
            snap = [t.clone() for t in state]
            bufs = [b.clone() for b in self.model.buffers()]
            seed = RT._seed_t.clone() if RT._seed_t is not None else None
            side = self._capture_stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._update(static_samples)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            with torch.no_grad():
                for t, s in zip(state, snap):
                    t.copy_(s)
                for b, s in zip(self.model.buffers(), bufs):
                    b.copy_(s)
                if seed is not None:
                    RT._seed_t.copy_(seed)
            RT.invalidate_shadows()
            self._sharded_dirty = False
            self._warmed = True
        # a cache miss later on captures directly: capture executes nothing (no state change, no collective runs)
        graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        # warm-up and every capture run on ONE side stream: autograd binds a parameter's AccumulateGrad node to the stream
        # of the forward that created it, and a node that survives an iteration (the speech-input path keeps some alive)
        # on a different stream than the capturing one forks the capture ("capturing stream has unjoined work")
        with torch.cuda.graph(graph, stream=self._capture_stream()):
            static_out = self._update(static_samples)
        torch.cuda.synchronize()
        ent = (graph, static_samples, static_out, static_flat)
        self._graphs[sig] = ent
        while len(self._graphs) > self.graph_cache_size:
            self._graphs.popitem(last=False)
        return ent

    def valid_step(self, sample):
        """tasks/speecht5.py:558-571 through the device path (eval mode, no gradient). With sharded training the bf16
        shadows are complete on every rank; parity mode additionally needs `consolidate()`."""
        if RT.dtype == torch.float32:
            self.consolidate()
        for c in (getattr(self.criterion, "text_to_speech_loss", None), getattr(self.criterion, "speech_to_text_loss", None)):
            if c is not None:
                c.defer_logging = False
        RT.layer_keep = None
        return self.task.valid_step(_to_device(sample, self.device), self.model, self.criterion)


# ---------------------------------------------------------------------------------------------------- batch plumbing
def pad_to_buckets(sample, buckets):
    """Pad the time axes of a collated batch to bucket multiples so that few distinct shapes (= captured graphs) occur:
    text tokens with the pad id, frames / waveform samples with zeros. Lengths and masks are untouched, so the criterion
    sees the same valid region (data/text_to_speech_dataset.py:223-281, data/speech_to_text_dataset.py:150-204).
    buckets: {"text": m, "frames": m (a multiple of the reduction factor), "wave": m, "target": m}."""
    def up(n, m):
        return (n + m - 1) // m * m

    def pad_dim(t, dim, to, value):
        if t.size(dim) == to:
            return t
        shape = list(t.shape)
        shape[dim] = to - t.size(dim)
        return torch.cat([t, t.new_full(shape, value)], dim=dim)
    out = dict(sample)
    ni = dict(sample["net_input"])
    task = sample.get("task_name", ni.get("task_name"))
    if task == "t2s":
        if "text" in buckets:
            ni["src_tokens"] = pad_dim(ni["src_tokens"], 1, up(ni["src_tokens"].size(1), buckets["text"]), 1)
        if "frames" in buckets:
            r = max(1, sample["dec_target"].size(1) // max(1, ni["prev_output_tokens"].size(1)))
            L = up(sample["dec_target"].size(1), buckets["frames"])
            out["dec_target"] = pad_dim(sample["dec_target"], 1, L, 0.0)
            out["labels"] = pad_dim(sample["labels"], 1, L, 0.0)
            ni["prev_output_tokens"] = pad_dim(ni["prev_output_tokens"], 1, L // r, 0.0)
            # the collater's padded features (data/text_to_speech_dataset.py:250-262; only their batch size is read):
            # left at their raw length they made every raw shape its own graph signature
            if torch.is_tensor(sample.get("target")) and sample["target"].dim() == 3:
                out["target"] = pad_dim(sample["target"], 1, up(sample["target"].size(1), buckets["frames"]), 0.0)
    elif task == "s2t":
        if "wave" in buckets:
            n = up(ni["source"].size(1), buckets["wave"])
            ni["source"] = pad_dim(ni["source"], 1, n, 0.0)
            if ni.get("padding_mask") is not None:
                ni["padding_mask"] = pad_dim(ni["padding_mask"], 1, n, True)
        if "target" in buckets:
            n = up(sample["target"].size(1), buckets["target"])
            out["target"] = pad_dim(sample["target"], 1, n, 1)
            ni["prev_output_tokens"] = pad_dim(ni["prev_output_tokens"], 1, n, 1)
    out["net_input"] = ni
    return out


def _flatten(sample, prefix=""):
    out = {}
    for k, v in sample.items():
        if isinstance(v, dict):
            out.update(_flatten(v, prefix + k + "."))
        elif torch.is_tensor(v):
            out[prefix + k] = v
    return out


def _to_device(sample, dev):
    if torch.is_tensor(sample):
        return sample.to(dev, non_blocking=True)
    if isinstance(sample, dict):
        return {k: _to_device(v, dev) for k, v in sample.items()}
    if isinstance(sample, (list, tuple)):  # (target_list of the pre-training collater, speech_dataset.py:383-385)
        return type(sample)(_to_device(v, dev) for v in sample)
    return sample


def _to_device_packed(samples, dev):
    """Device copies of a list of micro-batches whose tensors are views of ONE byte buffer (every tensor 256-byte
    aligned): a second set made the same way can be moved over it with a single device->device copy. Returns
    (list of dicts with the samples' structure, the byte buffer)."""
    sizes, total = [], 0
    for s in samples:
        for v in _flatten(s).values():
            n = v.numel() * v.element_size()
            sizes.append((total, n))
            total += (n + 255) // 256 * 256
    flat = torch.empty(max(total, 256), dtype=torch.uint8, device=dev)
    it = iter(sizes)

    def build(x):
        if torch.is_tensor(x):
            off, n = next(it)
            view = flat[off:off + n].view(x.dtype).view(x.shape)
            view.copy_(x, non_blocking=True)
            return view
        if isinstance(x, dict):
            return {k: build(v) for k, v in x.items()}
        return x
    return [build(s) for s in samples], flat


def _copy_into(static, new):
    for k, v in new.items():
        if isinstance(v, dict):
            _copy_into(static[k], v)
        elif torch.is_tensor(v):
            static[k].copy_(v, non_blocking=True)


def h2d_bytes(sample):
    if torch.is_tensor(sample):
        return sample.numel() * sample.element_size()
    if isinstance(sample, dict):
        return sum(h2d_bytes(v) for v in sample.values())
    if isinstance(sample, (list, tuple)):
        return sum(h2d_bytes(v) for v in sample)
    return 0
