"""CUDA-graph capture of one training step -- forward + loss (+ per-step accuracy) + backward [+ gradient all-reduce]
[+ fused optimizer] -- of the drop-in networks.

The hot path is ~150 short kernel launches per step issued from Python through ctypes; at a roofline step time of
~0.5 ms the launch path would dominate.  ``GraphedStep`` captures the launches once (static shapes, static input /
output buffers) and replays them with one ``cudaGraphLaunch`` -- "CUDA streams and graphs instead of a tracing
compiler".

    step = GraphedStep(model, lossfn, x_example, y_example, optimizer=FusedAdamW(model.parameters(), lr=1e-3))
    loss = step(x, y)            # copies x, y into the static buffers, replays, returns the loss tensor
    step.prefetch(x2, y2); loss = step(prefetched=True)   # pipelined form: the H2D copy overlaps the previous step
    step.dice                    # the reference's per-step accuracy (model/metric.py) from the SAME loss pass
    # model.parameters() .grad hold this step's gradients (static tensors, overwritten per replay)

The step drives the layer program (``engine.Engine``) directly -- the same kernels in the same order as the
``model(x) -> lossfn(logits, y) -> loss.backward()`` autograd path (``tests/test_engine_cpu.py`` and the GPU suite
check that both give the same loss and gradients) -- which lets it skip what nobody reads in a training step (the
fp32 ``probs`` tensor: the accuracy comes from the loss pass) and put the collectives where they overlap.

Data parallel (``enable_data_parallel()`` active; SURVEY.md 8e): the loss partial sums are all-reduced between the
loss pass and its finalize (global-batch-exact Dice), and the flat gradient bucket is SUM-all-reduced in two pieces:
everything from the deepest encoder block to the head (96 % of the bytes; complete when ~40 % of the backward is
done) starts its all-reduce right there and overlaps the rest of the backward, the remainder follows at the end
(eager mode and the one-graph mode).  By default the collectives stay BETWEEN the graphs of a captured step (forward +
loss sums | all-reduce | backward | all-reduce | optimizer).  ``B200SEG_NCCL_IN_GRAPH=1`` captures the NCCL kernels
INSIDE one graph (thread-local capture mode, so the NCCL watchdog thread cannot invalidate the capture); tearing the
process group down while such a graph is alive can hang (torch 2.11 / NCCL 2.28), so it is opt-in.
"""
from __future__ import annotations

import os
from typing import Optional

import torch

from . import runtime
from .engine import Engine
from .losses import LOVASZ, SS, ignore_label, loss_spec, lovasz_check, lovasz_scale_size, prepare_labels


def _is_fused_optimizer(opt) -> bool:
    from .optim import _FusedAdamBase
    return isinstance(opt, _FusedAdamBase)


class GraphedStep:
    def __init__(self, model: torch.nn.Module, lossfn, x: torch.Tensor, y: torch.Tensor, warmup: int = 2,
                 optimizer: Optional[torch.optim.Optimizer] = None, use_graph: bool = True,
                 want_probs: bool = False):
        self.model, self.lossfn, self.optimizer = model, lossfn, optimizer
        self.want_probs = want_probs
        self.x = torch.empty_like(x)
        self.x.copy_(x)
        c = model.numclass if hasattr(model, "numclass") else model.out_channels
        y0 = prepare_labels(y, c)
        self.y = torch.empty_like(y0)
        self.y.copy_(y0)
        self.ncls = c
        self.dp, self.group = runtime.dp_state()
        self.use_graph = use_graph and x.is_cuda
        self.graphs = []             # [(graph, eager callable to run after it or None)]
        self._terms, self._alpha, self._gamma, self._alpha_f = loss_spec(lossfn)
        if self._terms == LOVASZ:
            lovasz_check(c)
            self._per_image, self._ignore = bool(lossfn.per_image), ignore_label(lossfn.ignore)
        dev = self.x.device
        self._one = torch.ones(1, dtype=torch.float32, device=dev)
        # class weights of the loss: a constant of the step, created once (not a fill launch inside every step)
        self._alpha_t = torch.ones(c, dtype=torch.float32, device=dev) if self._alpha is None else \
            torch.as_tensor(self._alpha, dtype=torch.float32, device=dev)
        self._fused_opt = optimizer is not None and _is_fused_optimizer(optimizer)
        if self._fused_opt:
            optimizer.prepare()
        self._plan = None
        if model.training and model.dropout_masks is None and x.is_cuda and runtime._TEST_BACKEND is None:
            self._plan = model.mask_plan(x.shape[0], dev)
        self._works = []
        self.loss = self.dice = self.probs = None
        for _ in range(max(1, warmup)):
            self._eager_step()
        if self.use_graph:
            self._capture()

    # ------------------------------------------------------------------ the step, in pieces
    def _masks(self):
        m = self.model
        if self._plan is not None:
            return self._plan.launch()               # seed/offset were handed to the device by _pre()
        return m._draw_masks(self.x)

    def _pre(self):
        """host-side work of a step that must stay OUTSIDE a capture: the generator bookkeeping of the masks"""
        if self._plan is not None and self.model.training:
            self._plan.refresh()

    def _a(self):
        """dropout masks + forward + loss partial sums (+ accuracy sums)"""
        m = self.model
        be = runtime.get_backend(self.x)
        eng = Engine(be, runtime.act_dtype(), m._dims)
        eng.want_probs = self.want_probs
        P = dict(zip(m._pnames, [p.detach() for _, p in m.named_parameters()]))
        masks = self._masks() if m.training else None
        x = self.x if self.x.dtype == torch.float32 else self.x.float()
        out = getattr(eng, m._arch + "_forward")(P, x, masks, True)
        self._cls = isinstance(out, torch.Tensor)
        if self._cls:
            # classifier: (N, C) logits, a volume of one voxel per sample for the loss kernels (losses.prepare_logits)
            logits, probs = out, None
            z = logits.view(logits.shape[0], 1, 1, 1, logits.shape[1])
        else:
            logits, probs = out
            perm = (0, 2, 3, 4, 1) if logits.dim() == 5 else (0, 2, 3, 1)
            z = logits.permute(*perm)
        if not z.is_contiguous():
            z = z.contiguous()
        c, n = z.shape[-1], z.shape[0]
        buf = torch.zeros(be.part_size(c) + n * c * 3, dtype=torch.float64, device=z.device)
        part, metric = buf[:be.part_size(c)], buf[be.part_size(c):].view(n, c, 3)
        if self._terms == SS:
            be.loss_partials_ss(z, self.y, part, metric)
        else:
            be.loss_partials(z, self.y, self._gamma, self._alpha_f, part, metric)
        acc = torch.empty(2, dtype=torch.float32, device=z.device)
        be.metric_finalize(metric, acc)
        self._eng, self._z, self._part, self.probs, self._acc = eng, z, part, probs, acc
        self.dice = acc[0]

    def _ar_part(self):
        if self.dp:
            import torch.distributed as dist
            dist.all_reduce(self._part, op=dist.ReduceOp.SUM, group=self.group)      # SURVEY.md 8e (C2)

    def _bucket_ready(self, flat: torch.Tensor, off: int):
        """engine callback: gradients flat[off:] are final -> start their all-reduce now (overlaps the rest of backward)"""
        if self.dp and self._overlap:
            import torch.distributed as dist
            self._split_off = off
            self._works.append(dist.all_reduce(flat[off:], op=dist.ReduceOp.SUM, group=self.group, async_op=True))

    def _b(self):
        """loss finalize + d loss / d logits + network backward -> flat gradient bucket"""
        be = runtime.get_backend(self.x)
        z, part, eng = self._z, self._part, self._eng
        c = z.shape[-1]
        dev = z.device
        loss = torch.empty((), dtype=torch.float32, device=dev)
        dz = torch.empty_like(z)
        if self._terms == LOVASZ:
            coef = torch.empty_like(z)
            scale = torch.empty(lovasz_scale_size(z.shape[0], c, self._per_image), dtype=torch.float32, device=dev)
            be.lovasz_fwd(z, self.y, self._per_image, self._ignore, loss, coef, scale)
            be.lovasz_bwd(z, self.y, self._per_image, coef, scale, self._one, dz)
        else:
            lcoef = torch.empty(2 * c + 3 if c > 1 else 5, dtype=torch.float32, device=dev)
            be.loss_finalize(part, c, self._terms, self._alpha_t, self._gamma, self._alpha_f, loss, lcoef)
            if self._terms == SS:
                be.loss_bwd_ss(z, self.y, lcoef, self._one, dz)
            else:
                be.loss_bwd(z, self.y, lcoef, self._one, dz)
        if self._cls:
            g = dz.view(dz.shape[0], c)
        else:
            g = dz if dz.dim() == 5 else dz.unsqueeze(1)
        self._split_off = None
        eng.bucket_hook = self._bucket_ready if self.dp else None
        flat = getattr(eng, self.model._arch + "_backward")(g)
        self.loss, self._flat = loss, flat
        self._grads = [eng.grads[n] for n in self.model._pnames]

    def _ar_flat(self):
        if not self.dp:
            return
        import torch.distributed as dist
        if self._split_off is not None:
            if self._split_off > 0:
                dist.all_reduce(self._flat[:self._split_off], op=dist.ReduceOp.SUM, group=self.group)
            for w in self._works:
                w.wait()
            self._works = []
        else:
            dist.all_reduce(self._flat, op=dist.ReduceOp.SUM, group=self.group)      # SURVEY.md 8e (C1)

    def _c(self):
        """fused optimizer step on the flat bucket (one launch); torch optimizers run eagerly in _post()"""
        if self._fused_opt:
            self.optimizer.step(flat_grad=self._flat)

    def _post(self):
        for p, g in zip(self.model.parameters(), self._grads):
            if p.grad is not g:
                p.grad = g                      # also after a user's zero_grad(set_to_none=True)
        if self.optimizer is not None and not self._fused_opt:
            self.optimizer.step()

    def _eager_step(self):
        self._overlap = True
        with torch.no_grad():
            self._pre()
            self._a()
            self._ar_part()
            self._b()
            self._ar_flat()
            self._c()
        self._post()
        return self.loss

    # ------------------------------------------------------------------ capture
    def _capture(self):
        torch.cuda.synchronize()
        # B200SEG_HIPRI=1 captures the chain forward -> loss -> data gradients on a high-priority stream (the weight
        # gradients run beside it on the engine's default-priority side stream).  The persistent weight-gradient kernels
        # are then starved to the end of the step instead of filling the gaps of the chain, so it is off by default.
        hp = None
        if os.environ.get("B200SEG_HIPRI", "0") == "1":
            hp = torch.cuda.Stream(device=self.x.device, priority=-1)
        kw = {"stream": hp} if hp is not None else {}
        in_graph = self.dp and os.environ.get("B200SEG_NCCL_IN_GRAPH", "0") == "1"
        if not self.dp or in_graph:
            try:
                g = torch.cuda.CUDAGraph()
                self._overlap = True
                with torch.no_grad():
                    with torch.cuda.graph(g, capture_error_mode="thread_local" if self.dp else "global", **kw):
                        self._a()
                        self._ar_part()
                        self._b()
                        self._ar_flat()
                        self._c()
                self.graphs = [(g, None)]
            except Exception as e:                                  # noqa: BLE001
                if not self.dp:
                    raise
                import sys
                print(f"[b200seg] NCCL inside the step graph failed ({type(e).__name__}: {e}); "
                      "collectives stay between three graphs", file=sys.stderr)
                torch.cuda.synchronize()
                self._works = []
                self.graphs = []
        if not self.graphs:
            # collectives between the graphs (no overlap of the gradient all-reduce with the backward)
            self._overlap = False
            ga, gb, gc = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.no_grad():
                with torch.cuda.graph(ga, **kw):
                    self._a()
                self._ar_part()
                with torch.cuda.graph(gb, pool=ga.pool(), **kw):
                    self._b()
                self._ar_flat()
                self.graphs = [(ga, self._ar_part), (gb, self._ar_flat)]
                if self._fused_opt:
                    with torch.cuda.graph(gc, pool=ga.pool(), **kw):
                        self._c()
                    self.graphs.append((gc, None))
        torch.cuda.synchronize()
        self._post_bind()

    def _post_bind(self):
        for p, g in zip(self.model.parameters(), self._grads):
            p.grad = g

    @property
    def graph(self):
        """the step graph when the whole step is ONE graph (single GPU, or NCCL captured inside), else None"""
        return self.graphs[0][0] if len(self.graphs) == 1 else None

    # ------------------------------------------------------------------ input prefetch
    def prefetch(self, x: torch.Tensor, y: torch.Tensor) -> None:
        """Start the host->device copy of the NEXT step's inputs on a copy stream (pinned host tensors) while the
        current step is still running; ``step(prefetched=True)`` then only moves them device-to-device into the
        static buffers.  This is the input pipeline a training loop would run around the graph."""
        if not self.x.is_cuda:
            self._staged_host = (x, y)
            return
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(device=self.x.device)
            self._sx, self._sy = torch.empty_like(self.x), torch.empty_like(self.y)
            self._staged_ev = torch.cuda.Event()
            self._free_ev = torch.cuda.Event()
            self._free_ev.record(torch.cuda.current_stream(self.x.device))
        cs = self._copy_stream
        cs.wait_event(self._free_ev)                 # the previous step has drained the staging buffers
        with torch.cuda.stream(cs):
            self._sx.copy_(x, non_blocking=True)
            self._sy.copy_(y, non_blocking=True)
            self._staged_ev.record(cs)

    def _take_prefetched(self) -> None:
        if not self.x.is_cuda:
            x, y = self._staged_host
            self.x.copy_(x)
            self.y.copy_(y)
            return
        main = torch.cuda.current_stream(self.x.device)
        main.wait_event(self._staged_ev)
        self.x.copy_(self._sx, non_blocking=True)
        self.y.copy_(self._sy, non_blocking=True)
        self._free_ev.record(main)

    # ------------------------------------------------------------------ replay
    def __call__(self, x: Optional[torch.Tensor] = None, y: Optional[torch.Tensor] = None,
                 prefetched: bool = False) -> torch.Tensor:
        if prefetched:
            self._take_prefetched()
        if x is not None:
            self.x.copy_(x, non_blocking=True)
        if y is not None:
            self.y.copy_(y, non_blocking=True)
        if not self.graphs:
            return self._eager_step()
        self._pre()
        for g, after in self.graphs:
            g.replay()
            if after is not None:
                after()
        self._post()
        return self.loss

    def check_labels(self) -> None:
        """Raise if the last step saw a label outside [0, numclass) (the reference raises in F.one_hot /
        F.cross_entropy; a captured step cannot, so the loss becomes NaN and this check names the cause).
        Synchronises.  LovaszLoss takes such labels as background (the reference does not raise there)."""
        if self.ncls > 1 and self._terms != LOVASZ:
            bad = int(self._part[-1].item())
            if bad:
                raise RuntimeError(f"{bad} label value(s) outside [0, {self.ncls})")
