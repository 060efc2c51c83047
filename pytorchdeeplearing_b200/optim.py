"""Fused optimizer step of the training loop (SURVEY.md 8f-1): ``optim.AdamW(self.model.parameters(), lr=lr)``
(reference model/modelVNet.py:548; ``optim.Adam`` at model/modelUnet.py:849) as ONE sm_90a kernel launch over flat
fp32 parameter / gradient / moment buffers (``b200seg_adam_step``) instead of ~6 foreach launches over 128 tensors.

    opt = FusedAdamW(model.parameters(), lr=1e-3)        # same constructor arguments as torch.optim.AdamW
    opt.zero_grad(); loss.backward(); opt.step()         # the reference's loop, unchanged (modelVNet.py:590-593)

On first use the parameters are re-homed into ONE flat buffer (``p.data`` become views: ``state_dict`` /
``load_state_dict`` / the kernels see no difference).  When the gradients are views of the engine's flat bucket at
the matching offsets (they are after ``loss.backward()`` / ``GraphedStep``), the whole update is one launch; otherwise
the same kernel runs once per parameter.  The step count lives on the device, so the update can be captured in a CUDA
graph (``GraphedStep(optimizer=FusedAdamW(...))``) and replayed.
"""
from __future__ import annotations

from typing import List

import torch

from . import runtime


class _FusedAdamBase(torch.optim.Optimizer):
    _decoupled = False

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        if lr < 0 or eps < 0 or weight_decay < 0 or not 0 <= betas[0] < 1 or not 0 <= betas[1] < 1:
            raise ValueError("invalid optimizer hyper-parameter")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._flat = {}          # group index -> dict(param, exp_avg, exp_avg_sq, state, offsets)

    # ------------------------------------------------------------------ flat state
    def _flatten(self, gi: int, group):
        ps: List[torch.Tensor] = [p for p in group["params"] if p.requires_grad]
        if not ps:
            return None
        dev = ps[0].device
        for p in ps:
            if p.dtype != torch.float32 or p.device != dev:
                raise RuntimeError("FusedAdam needs fp32 parameters on one device")
        total = sum(p.numel() for p in ps)
        flat = torch.empty(total, dtype=torch.float32, device=dev)
        offs, off = [], 0
        for p in ps:
            view = flat[off:off + p.numel()].view(p.shape)
            view.copy_(p.data)                       # re-home the parameter: p.data is a view of the flat buffer
            p.data = view
            offs.append(off)
            off += p.numel()
        st = dict(params=ps, flat=flat, offs=offs, total=total,
                  exp_avg=torch.zeros(total, dtype=torch.float32, device=dev),
                  exp_avg_sq=torch.zeros(total, dtype=torch.float32, device=dev),
                  state=torch.zeros(4, dtype=torch.float32, device=dev))
        self._flat[gi] = st
        return st

    def _still_flat(self, st) -> bool:
        base = st["flat"].data_ptr()
        return all(p.data_ptr() == base + 4 * o for p, o in zip(st["params"], st["offs"]))

    def prepare(self):
        """Flatten now (e.g. before capturing a step) instead of at the first ``step()``."""
        for gi, group in enumerate(self.param_groups):
            if gi not in self._flat:
                self._flatten(gi, group)
        return self

    # ------------------------------------------------------------------ step
    @torch.no_grad()
    def step(self, closure=None, flat_grad: torch.Tensor = None):
        """``flat_grad``: the engine's flat gradient bucket (parameter order) when the caller has it at hand
        (GraphedStep); otherwise the ``.grad`` of the parameters are used."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for gi, group in enumerate(self.param_groups):
            st = self._flat.get(gi)
            if st is None or not self._still_flat(st):
                st_old = st
                st = self._flatten(gi, group)            # (re-)home, e.g. after model.to(device)
                if st is None:
                    continue
                if st_old is not None and st_old["total"] == st["total"]:
                    for k in ("exp_avg", "exp_avg_sq", "state"):
                        st[k].copy_(st_old[k])
            be = runtime.get_backend(st["flat"])
            b1, b2 = group["betas"]
            hyper = (float(group["lr"]), float(b1), float(b2), float(group["eps"]), float(group["weight_decay"]),
                     self._decoupled)
            ps, offs = st["params"], st["offs"]
            fg = flat_grad
            if fg is None:
                grads = [p.grad for p in ps]
                if any(g is None for g in grads):
                    if all(g is None for g in grads):
                        continue
                    raise RuntimeError("FusedAdam: some parameters have no gradient (all or none must take part)")
                g0 = grads[0].data_ptr() - 4 * offs[0]
                if all(g.dtype == torch.float32 and g.is_contiguous() and g.data_ptr() == g0 + 4 * o
                       for g, o in zip(grads, offs)):
                    # gradients already form one flat buffer in parameter order (engine bucket): ONE launch
                    fg = torch.as_strided(grads[0].reshape(-1), (st["total"],), (1,),
                                          storage_offset=grads[0].storage_offset() - offs[0])
            if fg is not None:
                if fg.numel() != st["total"] or fg.dtype != torch.float32:
                    raise RuntimeError("FusedAdam: flat gradient does not match the parameters")
                be.adam_step(st["flat"], fg, st["exp_avg"], st["exp_avg_sq"], st["state"], *hyper)
            else:
                first = True
                for p, o in zip(ps, offs):
                    n = p.numel()
                    g = p.grad if p.grad.is_contiguous() and p.grad.dtype == torch.float32 else \
                        p.grad.float().contiguous()
                    be.adam_step(st["flat"][o:o + n], g.reshape(-1), st["exp_avg"][o:o + n],
                                 st["exp_avg_sq"][o:o + n], st["state"], *hyper, tick=first)
                    first = False
        return loss


class FusedAdamW(_FusedAdamBase):
    """torch.optim.AdamW semantics (decoupled weight decay, default 0.01) -- model/modelVNet.py:548."""
    _decoupled = True

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2):
        super().__init__(params, lr, betas, eps, weight_decay)


class FusedAdam(_FusedAdamBase):
    """torch.optim.Adam semantics (L2 weight decay folded into the gradient, default 0) -- model/modelUnet.py:849."""
    _decoupled = False


__all__ = ["FusedAdamW", "FusedAdam"]
