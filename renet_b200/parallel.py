"""Data parallelism for the hot path (SURVEY.md section 8(e)): one process per GPU, every rank runs the whole
RGCN-aggregate + GRU path on its own slice of the global batch (its own batched history graph -- components may
repeat across ranks, which is cheaper than exchanging them), parameters replicated, the gradient all-reduced
(NCCL over NVLink on the GPUs; gloo on CPU for the tests) in buckets that are launched from autograd hooks WHILE the
backward kernels of the remaining layers still run, then clip-grad-norm on the reduced gradient (reference
train.py:140) and Adam (train.py:61,141).

The reference itself is single-GPU (train.py:33); nothing here has a reference counterpart except the step
sequence of train.py:136-143, which ``DataParallelTrainer.train_step`` follows.

Layout: every trainable parameter is re-pointed into ONE flat fp32 buffer (``flat_p``) and its ``.grad`` into a
second one (``flat_g``), in reverse registration order (roughly the order gradients become ready in backward, as in
torch DDP).  Buckets are contiguous ranges of ``flat_g``, so a bucket's all-reduce needs no packing copy, the
bucket list is identical on every rank by construction (parameters without a gradient on some rank simply
contribute zeros), and the optimiser step is two launches over the flat buffers (csrc/optim.cu).
"""
import numpy as np
import torch
import torch.distributed as dist

from . import _lib

ALIGN = 64        # floats: every parameter starts on a 256-byte boundary of the flat buffers


def shard_slice(n, rank, world):
    """[lo, hi) of rank's contiguous slice of n items (global batch 8192 -> 8 x 1024)."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_batch(batch, s_hist, o_hist, rank, world):
    """Slice (triplets, (s_hist, s_hist_t), (o_hist, o_hist_t)) of a GLOBAL batch for this rank."""
    lo, hi = shard_slice(len(batch), rank, world)
    cut = lambda pair: (pair[0][lo:hi], pair[1][lo:hi])
    return batch[lo:hi], cut(s_hist), cut(o_hist), (hi - lo)


def round_robin(n_units, rank, world):
    """The units of rank when n_units are handed out round-robin -- unit c to rank c mod world -- in unit order."""
    return range(rank, n_units, world)


class Shard:
    """One process's place in an evaluation sharded over ``group`` (RENet.evaluate_stream_batched(process_group=...)):
    its rank and the group's size, and the exchanges the sharded units need.  Exchanges run on ``device`` over NCCL and on
    the host over any other backend; their results come back on the device of what was sent."""

    def __init__(self, group, device):
        self.group = group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.xdev = torch.device(device) if dist.get_backend(group) == 'nccl' else torch.device('cpu')

    def units(self, n_units):
        return round_robin(n_units, self.rank, self.world)

    def slice(self, n):
        return shard_slice(n, self.rank, self.world)

    def allgather(self, local, counts):
        """Every rank's block of rows, in rank order: ``local`` [counts[rank], ...] is this rank's, ``counts`` every rank's
        row count (known on every rank).  The blocks travel padded to the largest one."""
        cap = max(counts)
        if cap == 0:
            return [local[:0]] * self.world
        buf = torch.zeros((cap,) + tuple(local.shape[1:]), dtype=local.dtype, device=self.xdev)
        buf[:len(local)] = local
        out = [torch.empty_like(buf) for _ in range(self.world)]
        dist.all_gather(out, buf, group=self.group)
        return [o[:c].to(local.device) for o, c in zip(out, counts)]

    def allgather_slices(self, local, n):
        """The whole of n rows on every rank, from each rank's contiguous slice(n) of them, ``local`` being this rank's."""
        counts = [hi - lo for lo, hi in (shard_slice(n, r, self.world) for r in range(self.world))]
        return torch.cat(self.allgather(local, counts))

    def gather_units(self, blocks, sizes, empty):
        """Every unit's block, in unit order, on every rank.  ``sizes[c]`` is unit c's row count; ``blocks`` are the blocks of
        this rank's units (units(len(sizes)), in order); ``empty`` is a zero-row tensor of the blocks' trailing shape, dtype
        and device."""
        n = len(sizes)
        counts = [sum(sizes[c] for c in round_robin(n, r, self.world)) for r in range(self.world)]
        got = self.allgather(torch.cat([empty] + list(blocks)), counts)
        out = [None] * n
        for r in range(self.world):
            off = 0
            for c in round_robin(n, r, self.world):
                out[c] = got[r][off:off + sizes[c]]
                off += sizes[c]
        return out

    def same_everywhere(self, values):
        """True when the int64 vector ``values`` is the same on every rank (one small all-gather; the answer is the same on
        every rank)."""
        v = torch.as_tensor(values, dtype=torch.long).view(1, -1)
        got = self.allgather(v, [1] * self.world)
        return all(torch.equal(g, got[0]) for g in got)


def _world(group=None):
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(group)
    return 1


def allreduce_gradients(params, local_weight=1.0, bucket_bytes=64 << 20, group=None):
    """One-shot weighted gradient average over ranks for an arbitrary parameter list (no hooks, no flat views):
    used by callers that keep their own optimiser.  Buckets are built over the FULL parameter list, which is the
    same on every rank; a parameter whose gradient is missing on this rank contributes zeros (and receives the
    average), so the collective sizes can never differ between ranks."""
    world = _world(group)
    params = list(params)
    if world == 1 or not params:
        return
    dev = params[0].device
    w = torch.tensor([float(local_weight)], device=dev, dtype=torch.float32)
    dist.all_reduce(w, group=group)
    scale = float(local_weight) / float(w.item())
    buckets, cur, cur_bytes = [], [], 0
    for p in params:
        nb = p.numel() * p.element_size()
        if cur and cur_bytes + nb > bucket_bytes:
            buckets.append(cur); cur, cur_bytes = [], 0
        cur.append(p); cur_bytes += nb
    if cur:
        buckets.append(cur)
    pending = []
    for b in buckets:
        flat = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in b]).mul_(scale)
        pending.append((b, flat, dist.all_reduce(flat, group=group, async_op=True)))
    for b, flat, work in pending:
        work.wait()
        off = 0
        for p in b:
            n = p.numel()
            if p.grad is None:
                p.grad = flat[off:off + n].view_as(p).clone()
            else:
                p.grad.copy_(flat[off:off + n].view_as(p))
            off += n


def native_optimizer_step(tr):
    """clip_grad_norm_ + Adam on the flat buffers through librenet_b200.so (CUDA only; no fallback)."""
    _lib.require_cuda(tr.flat_p, tr.flat_g)
    L = _lib.lib()
    P = _lib.ptr
    st = _lib.stream()
    n = tr.flat_p.numel()
    sumsq = None
    if tr.grad_norm is not None and tr.grad_norm > 0:
        _lib.check(L.renet_grad_sumsq(P(tr.flat_g), n, P(tr._sumsq), 0, P(tr._red_ws), tr._red_ws.numel() * 4, st),
                   'renet_grad_sumsq')
        sumsq = tr._sumsq
    _lib.check(L.renet_adam_step(P(tr.flat_p), P(tr.flat_g), P(tr.exp_avg), P(tr.exp_avg_sq), n, tr.lr, tr.betas[0],
                                 tr.betas[1], tr.eps, tr.weight_decay, tr.step_count, P(sumsq),
                                 float(tr.grad_norm or 0.0), 1.0, st), 'renet_adam_step')
    _lib.invalidate_packed_weights()          # the update went through raw pointers: p._version did not move


class DataParallelTrainer:
    """Replicated-parameter data parallelism with bucketed gradient all-reduce overlapped with backward.

        tr = DataParallelTrainer(model, lr=1e-3, weight_decay=1e-5, grad_norm=1.0)
        loss = tr.train_step(batch, s_hist, o_hist, graph_dict)            # train.py:136-143 on this rank's shard

    ``optimizer_step`` (callable taking the trainer) replaces the native CUDA optimiser; the CPU/gloo tests pass a
    torch restatement.  Timing hooks: after ``step`` returns, ``last_events`` holds CUDA events (forward start,
    backward start, backward end, all-reduce drained, step end) when ``record_events`` is set."""

    def __init__(self, model, lr=1e-3, weight_decay=1e-5, betas=(0.9, 0.999), eps=1e-8, grad_norm=1.0,
                 bucket_bytes=25 << 20, group=None, optimizer_step=None, overlap=True, record_events=False):
        self.model, self.group = model, group
        self.lr, self.weight_decay, self.betas, self.eps, self.grad_norm = lr, weight_decay, betas, eps, grad_norm
        self.world = _world(group)
        self.overlap = overlap
        self.optimizer_step = optimizer_step or native_optimizer_step
        self.record_events = record_events
        self.last_events = None
        self.step_count = 0
        params = [p for p in model.parameters() if p.requires_grad]
        if not params:
            raise ValueError('DataParallelTrainer: the model has no trainable parameters')
        self.params = params[::-1]                        # ~ the order gradients become ready in backward
        dev, dt = params[0].device, params[0].dtype
        if dt != torch.float32 or any(p.dtype != dt or p.device != dev for p in params):
            raise ValueError('DataParallelTrainer: all parameters must be fp32 on one device')
        offs, o = [], 0
        for p in self.params:
            offs.append(o)
            o += (p.numel() + ALIGN - 1) // ALIGN * ALIGN
        self.offsets, self.total = offs, o
        self.flat_p = torch.zeros(o, device=dev)
        self.flat_g = torch.zeros(o, device=dev)
        self.exp_avg = torch.zeros(o, device=dev)
        self.exp_avg_sq = torch.zeros(o, device=dev)
        with torch.no_grad():
            for p, off in zip(self.params, offs):
                view = self.flat_p[off:off + p.numel()].view_as(p)
                view.copy_(p.data)
                p.data = view
                p.grad = self.flat_g[off:off + p.numel()].view_as(p)
        if dev.type == 'cuda':
            self._sumsq = torch.zeros(1, device=dev)
            self._red_ws = torch.empty(int(_lib.lib().renet_grad_sumsq_workspace_bytes()) // 4, device=dev)
        # buckets: contiguous ranges [lo, hi) of the flat gradient; a parameter never straddles two buckets
        self.buckets, cur_lo, cur_n = [], 0, []
        for i, (p, off) in enumerate(zip(self.params, offs)):
            end = off + (p.numel() + ALIGN - 1) // ALIGN * ALIGN
            if cur_n and (end - cur_lo) * 4 > bucket_bytes:
                self.buckets.append({'lo': cur_lo, 'hi': off, 'params': cur_n})
                cur_lo, cur_n = off, []
            cur_n.append(i)
        self.buckets.append({'lo': cur_lo, 'hi': o, 'params': cur_n})
        self._bucket_of = {}
        for b, bk in enumerate(self.buckets):
            for i in bk['params']:
                self._bucket_of[i] = b
        self._pending = [0] * len(self.buckets)
        self._launched = [None] * len(self.buckets)
        self._in_step = False
        self._next = 0
        self._hooks = [p.register_post_accumulate_grad_hook(self._make_hook(i)) for i, p in enumerate(self.params)]

    # ---- gradient exchange ------------------------------------------------------------------------------------
    def _make_hook(self, i):
        def hook(_p):
            if not self._in_step:
                return
            b = self._bucket_of[i]
            self._pending[b] -= 1
            if self.overlap:
                # collectives must be issued in the same order on every rank: bucket b goes out only after buckets 0..b-1
                # (a bucket that is complete early waits for its predecessors; one that never completes on this rank --
                # a parameter without gradient here -- goes out in _drain, still in order)
                while self._next < len(self.buckets) and self._pending[self._next] == 0:
                    self._launch(self._next)
        return hook

    def _launch(self, b):
        assert b == self._next
        self._next += 1
        if self.world == 1:
            return
        bk = self.buckets[b]
        self._launched[b] = dist.all_reduce(self.flat_g[bk['lo']:bk['hi']], group=self.group, async_op=True)

    def _drain(self):
        while self._next < len(self.buckets):    # buckets whose parameters got no gradient on this rank still take part
            self._launch(self._next)
        for b, w in enumerate(self._launched):
            if w is not None:
                w.wait()
            self._launched[b] = None

    def _ev(self):
        if self.record_events and self.flat_p.is_cuda:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            return e
        return None

    # ---- one optimisation step ---------------------------------------------------------------------------------
    def step(self, loss_fn, local_weight=None):
        """loss_fn() -> scalar loss of THIS rank's shard (a mean over its local samples, like nn.CrossEntropyLoss,
        model.py:57).  Gradients are averaged over ranks, weighted by ``local_weight`` (the local sample count) when
        given -- ragged last batch -- else uniformly.  A rank whose shard has no history at all (the reference crashes
        on such a batch, Aggregator.py:128-129) contributes a zero gradient instead of dropping out of the collective."""
        scale = 1.0 / self.world
        if local_weight is not None and self.world > 1:
            w = torch.tensor([float(local_weight)], device=self.flat_p.device)
            dist.all_reduce(w, group=self.group)
            scale = float(local_weight) / float(w.item())
        self._pending = [len(bk['params']) for bk in self.buckets]
        self._next = 0
        self._in_step = True
        evs = [self._ev()]
        try:
            try:
                loss = loss_fn()
            except ValueError as ex:
                if 'every history in the batch is empty' not in str(ex):
                    raise
                loss = None
            evs.append(self._ev())
            if loss is not None:
                (loss * scale if scale != 1.0 else loss).backward()
            evs.append(self._ev())
            self._drain()
            evs.append(self._ev())
        finally:
            self._in_step = False
        self.step_count += 1
        self.optimizer_step(self)
        evs.append(self._ev())
        self.last_events = evs if self.record_events else None
        return None if loss is None else loss.detach()

    def zero_grad(self):
        self.flat_g.zero_()

    def train_step(self, batch, s_hist, o_hist, graph_dict, local_weight=None):
        """One reference training step (train.py:136-143) on this rank's shard."""
        model = self.model

        def loss_fn():
            loss_s = model(batch, s_hist, o_hist, graph_dict, subject=True)
            loss_o = model(batch, s_hist, o_hist, graph_dict, subject=False)
            return loss_s + loss_o
        loss = self.step(loss_fn, local_weight)
        self.zero_grad()
        return loss

    def close(self):
        for h in self._hooks:
            h.remove()
        self._hooks = []


def train_step(model, optimizer, batch, s_hist, o_hist, graph_dict, grad_norm=1.0, local_weight=None):
    """One reference training step (train.py:136-143) with a caller-owned torch optimiser: backward, then ONE
    (non-overlapped) weighted gradient all-reduce, clip, step.  ``DataParallelTrainer`` is the fast path."""
    loss_s = model(batch, s_hist, o_hist, graph_dict, subject=True)
    loss_o = model(batch, s_hist, o_hist, graph_dict, subject=False)
    loss = loss_s + loss_o
    loss.backward()
    allreduce_gradients(list(model.parameters()), local_weight if local_weight is not None else len(batch))
    torch.nn.utils.clip_grad_norm_(model.parameters(), grad_norm)
    optimizer.step()
    optimizer.zero_grad()
    _lib.invalidate_packed_weights()
    return loss.detach()
