"""Layer program of the segmentation hot path (host side, Python).

The engine turns one forward/backward of ``VNet3d`` / ``UNet3d`` / ``UNet2d`` / ``ResNet3d`` into a sequence
of calls on a *backend* whose methods map 1:1 onto the ``extern "C"`` entry points of
``include/b200seg.h`` (``_abi.CudaBackend``).  It owns no arithmetic: every FLOP and every
byte moved happens inside a backend op (= one hand-written sm_90a kernel launch).

Data layout (DESIGN.md section 3): activations are channels-last ``(N, D, H, W, C)`` views
(2-D nets use ``D == 1``) with a channel pitch ``ld >= C`` so that producers write straight
into slices of a skip-concat buffer (``torch.cat`` of VNet3d.py:74 / Unet3d.py:45 is never
materialised).  Storage dtype ``T`` is bf16 (perf mode) or fp32 (parity mode); GroupNorm
statistics, loss partial sums and weight gradients are fp32/fp64.

Block algebra (SURVEY.md App. G): a ``conv -> GroupNorm(8) -> Dropout(p) -> ReLU`` block of
the reference (VNet3d.py:13-15, Unet3d.py:66-85) is executed as
  conv kernel (raw output y + per-(n,c) sum / sum-of-squares in the epilogue)
  -> gn_finalize (mean, rstd per (n,g); A = rstd*gamma*s, B = (beta - mean*rstd*gamma)*s per (n,c))
  -> apply      (act = relu(y*A + B) [+ second branch] [+ residual]), written where the consumer wants it.
"""
from __future__ import annotations

import os

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch

Tensor = torch.Tensor

# conv kinds understood by backend.conv / backend.wgrad
K3, K1, DOWN, UP = 0, 1, 2, 3
GROUPS = 8
GN_EPS = 1e-5
P_DROP = 0.2
ACT_RELU, ACT_LEAKY = 0, 1     # activation after the norm (B200SEG_ACT_*)


@dataclass(frozen=True)
class VNetSpec:
    """What distinguishes the VNet-shaped layer programs: LUConv ops per DownTransition / UpTransition (in pyramid
    order, up_tr256 first), the parameter names of the norms and the LUConv convolutions, the norm's groups (0: one
    per channel, InstanceNorm3d) and the activation."""
    down_ops: Tuple[int, ...] = (2, 3, 3, 3)
    up_ops: Tuple[int, ...] = (3, 3, 2, 1)
    in_bn: str = "bn1"          # in_tr.<in_bn>
    down_bn: str = "bn1"        # down_trX.<down_bn>
    op_conv: str = "conv1"      # X.ops.j.<op_conv>
    op_bn: str = "bn1"          # X.ops.j.<op_bn>
    groups: int = GROUPS
    act: int = ACT_RELU


VNET = VNetSpec()
# VNet3dRegistration (networks/VNet3dregistration.py:48-169): InstanceNorm3d(affine) and LeakyReLU(0.01)
REGISTRATION = VNetSpec(down_ops=(2, 2, 2, 2), up_ops=(2, 2, 2, 1), in_bn="bn", down_bn="bn", op_conv="conv",
                        op_bn="bn", groups=0, act=ACT_LEAKY)
# the ResNet stages whose outputs Grad-CAM can take (resnet_backward ``stages``), in forward order
RESNET_STAGES = ("in_tr", "down_tr32", "down_tr64", "down_tr128", "down_tr256")


@dataclass
class Layer:
    """One conv application (+ optional GroupNorm/Dropout/ReLU tail) and what backward needs."""
    kind: int
    wname: str
    bname: Optional[str]
    gname: Optional[str]            # GroupNorm prefix ("in_tr.bn1") or None
    x: Tensor = None                # input activation view (N,D,H,W,Cin)
    y: Tensor = None                # raw conv output (N,D',H',W',Cout)
    coef: Tensor = None             # (N,Cout,2) fp32  A,B          (unfused path only)
    mr: Tensor = None               # (N,G,2)   fp32  mean, rstd    (unfused path only)
    gn: tuple = None                # (stats, gamma, beta, scale, vox, groups, eps): fused-coefficient path
    scale: Optional[Tensor] = None  # (N,Cout) dropout scale or None
    pre_sums: Optional[Tensor] = None   # backward sums already accumulated by the epilogue of the conv that produced g
    wpk: object = None              # fused input block: packed forward operand of the stem (``y`` is never stored)


def _taps(kind: int, dims: int) -> int:
    if kind == K3:
        return 27 if dims == 3 else 9
    if kind == K1:
        return 1
    return 8 if dims == 3 else 4


# B200SEG_OVERLAP: bit mask of host-side scheduling options that move work off the serial kernel chain of a step onto
# the side stream (all of them launch the SAME kernels on the SAME data; only stream placement / launch grouping changes)
OV_PACK = 1      # forward: only the operands of the first block(s) are packed on the main stream; the rest of the
                 # step's pack launch runs on the side stream under the first convolutions
OV_UNPACK = 2    # backward: the weight gradients finished by the time the deepest encoder block is done (96 % of the
                 # bytes) are brought to parameter layout on the side stream there, not after the last kernel of the step
OV_TAIL = 4      # backward: the weight gradient of the first input-block branch runs beside the GroupNorm backward of
                 # the second one (neither has a data gradient behind it)
OV_ZERO = 8      # the zero fills backward needs (gradient bucket, accumulator arenas) are issued on the side stream
                 # during forward
OV_ALL = OV_PACK | OV_UNPACK | OV_TAIL | OV_ZERO


def overlap_mask(arch: str = "vnet", dims: int = 3) -> int:
    """``B200SEG_OVERLAP`` if set, else the default: all four options together for VNet3d / VNet2d / UNet2d on one GPU,
    the plain schedule for the 3-D UNets (UNet3d, UNet3dthin) and for data-parallel runs (``tools/overlap_ab.py`` is the
    A/B harness)."""
    e = os.environ.get("B200SEG_OVERLAP")
    if e is not None:
        try:
            return int(e) & OV_ALL
        except ValueError:
            return 0
    if arch in ("unet", "unetthin") and dims == 3:
        return 0
    from . import runtime
    if runtime.dp_state()[0]:
        return 0
    return OV_ALL


_SIDE_STREAMS: Dict[int, "torch.cuda.Stream"] = {}


def _side_stream(device) -> Optional["torch.cuda.Stream"]:
    """Second stream for the weight gradients (independent of the data-gradient chain once dy exists); joins the
    main stream again in ``_finish_backward``.  Works under CUDA-graph capture (fork/join become graph edges)."""
    if device.type != "cuda" or os.environ.get("B200SEG_WGRAD_SIDE_STREAM", "1") == "0":
        return None
    idx = device.index if device.index is not None else torch.cuda.current_device()
    st = _SIDE_STREAMS.get(idx)
    if st is None:
        st = _SIDE_STREAMS[idx] = torch.cuda.Stream(device=idx)
    return st


class _ZeroArena:
    """One zero-filled allocation per pass, handed out as views: replaces ~100 tiny fill launches per step
    (GroupNorm statistics, backward sums, split-K weight-gradient accumulators) by one memset each."""

    def __init__(self, dtype: torch.dtype, numel: int, device, buf: Optional[Tensor] = None):
        # ``buf``: an already zeroed (or being zeroed, on a stream the user joins) allocation of that size
        self.buf = torch.zeros(max(1, numel), dtype=dtype, device=device) if buf is None else buf
        self.off = 0

    def take(self, shape) -> Tensor:
        n = 1
        for s in shape:
            n *= s
        n_al = (n + 15) // 16 * 16                      # keep every view 128-byte aligned
        if self.off + n_al > self.buf.numel():
            return torch.zeros(shape, dtype=self.buf.dtype, device=self.buf.device)
        v = self.buf[self.off:self.off + n].view(shape)
        self.off += n_al
        return v


class Engine:
    """Executes the layer program on ``backend``.  ``P`` maps reference state_dict names to
    fp32 parameter tensors (App. A layout)."""

    def __init__(self, backend, act_dtype: torch.dtype, dims: int):
        self.be = backend
        self.T = act_dtype
        self.dims = dims
        self.P: Dict[str, Tensor] = {}
        self.masks: Optional[List[Tensor]] = None
        self._mi = 0
        self.layers: List[Layer] = []
        self.grads: Dict[str, Tensor] = {}
        self.saved: Dict[str, object] = {}
        self.need_grad = True
        self._z64 = None
        self._z32 = None
        self._packs: Dict[Tuple[str, str], object] = {}
        self._unpack_list: List[Tuple[Tensor, Tensor]] = []
        self.bucket_hook = None                # data parallel: callable(flat, offset) when flat[offset:] is final
        self._flat = None
        self._goff: Dict[str, int] = {}
        self.want_probs = True                 # False: the head writes logits only (GraphedStep: nobody reads probs)
        self.mask_threshold: Optional[float] = None   # not None: inference head -> uint8 mask, no logits / probs
        self._side = None                      # side stream carrying this pass's weight gradients (if any)
        self._side_keep: List[object] = []     # operands of side-stream kernels stay referenced until the join
        self._fwd_side = None                  # side stream carrying forward-time work (late pack, zero fills) not yet joined
        self._late: set = set()                # weights whose forward operand comes from the side-stream pack
        self._pre_bwd = None                   # (flat, z64 buffer, z32 buffer) zeroed during forward for backward
        self._deferred = None                  # (side, fork event, pack plan, zero buffers) not launched yet
        self._ov = 0                           # scheduling options of this pass (overlap_mask), fixed at forward
        self._data_only = False                # backward computes data gradients only (no weight-gradient convolutions)
        self.spec = VNET                       # norm groups and activation of conv_gn (vnet_forward sets its spec)

    # ---------------------------------------------------------------- allocation helpers
    def new(self, like: Tensor, sp: Sequence[int], c: int, dtype=None) -> Tensor:
        return torch.empty((like.shape[0],) + tuple(sp) + (c,), dtype=dtype or self.T, device=like.device)

    def zeros(self, shape, dtype, device) -> Tensor:
        arena = self._z64 if dtype == torch.float64 else (self._z32 if dtype == torch.float32 else None)
        if arena is not None and arena.buf.device == device:
            return arena.take(tuple(shape))
        return torch.zeros(shape, dtype=dtype, device=device)

    def _arena_sizes(self, n: int, backward: bool) -> Tuple[int, int]:
        gn_ch = sum(p.numel() for k, p in self.P.items() if p.dim() == 1 and k.endswith(".weight"))
        per = 3 if backward else 2
        wel = sum(p.numel() for p in self.P.values() if p.dim() > 1) if backward else 0
        return n * gn_ch * per * 2 + 64 * 40, wel + 16 * 64

    def _begin_pass(self, n: int, device, backward: bool) -> None:
        n64, n32 = self._arena_sizes(n, backward)
        pre = self._pre_bwd if backward else None
        self._z64 = _ZeroArena(torch.float64, n64, device, buf=pre[1] if pre is not None else None)
        if backward:
            self._z32 = _ZeroArena(torch.float32, n32, device, buf=pre[2] if pre is not None else None)
        else:
            self._z32 = None

    def _zero_ahead_alloc(self, n: int, device):
        """OV_ZERO: what backward wants zero-filled (flat gradient bucket, both accumulator arenas) is allocated during
        forward and filled on the side stream under the forward kernels (``_launch_deferred``)."""
        n64, n32 = self._arena_sizes(n, True)
        total = sum(p.numel() for p in self.P.values())
        return (torch.empty(total, dtype=torch.float32, device=device),
                torch.empty(max(1, n64), dtype=torch.float64, device=device),
                torch.empty(max(1, n32), dtype=torch.float32, device=device))

    def _next_mask(self) -> Optional[Tensor]:
        if self.masks is None:
            return None
        m = self.masks[self._mi]
        self._mi += 1
        return m

    def _prepack(self, specs, need_grad: bool, n_early: int = 0) -> None:
        """ONE launch packs every conv operand of the step (forward and data-gradient layouts).
        specs: [(wname, kind, vox_out, vox_in, needs_dgrad)].  With OV_PACK the forward operands of the first
        ``n_early`` specs are packed by a small launch on the main stream; everything else is packed by a second launch
        on the side stream, enqueued right AFTER the first convolution of the pass (so that convolution's CTAs are
        dispatched first and the pack fills what it leaves free) and joined at the first use of one of its operands."""
        reqs, keys, late_reqs, late_keys = [], [], [], []
        self._tag(None)
        ov = self._ov
        dev = self.P[specs[0][0]].device
        side = _side_stream(dev)
        # (without a side stream -- CPU test backend, B200SEG_WGRAD_SIDE_STREAM=0 -- the same launches stay on the main stream)
        split = bool(ov & OV_PACK) and 0 < n_early < len(specs) and hasattr(self.be, "pack_plan")
        for i, (wname, kind, vox_out, vox_in, dgrad) in enumerate(specs):
            early = not split or i < n_early
            (reqs if early else late_reqs).append((self.P[wname], kind, "fwd", self.T, self.dims, vox_out))
            (keys if early else late_keys).append((wname, "fwd"))
            if need_grad and dgrad:
                (late_reqs if split else reqs).append((self.P[wname], kind, "dgrad", self.T, self.dims, vox_in))
                (late_keys if split else keys).append((wname, "dgrad"))
        self._packs = dict(zip(keys, self.be.pack_many(reqs)))
        self._late, self._fwd_side, self._pre_bwd, self._deferred = set(), None, None, None
        plan = bufs = None
        if late_reqs:
            plan = self.be.pack_plan(late_reqs)                 # allocations now, launches deferred
            self._packs.update(zip(late_keys, plan.outs))
            self._late = {k[0] for k in late_keys if k[1] == "fwd"}
        if need_grad and (ov & OV_ZERO):
            bufs = self._pre_bwd = self._zero_ahead_alloc(self._batch, dev)
        if plan is not None or bufs is not None:
            fork = None
            if side is not None:
                fork = torch.cuda.Event()
                fork.record(torch.cuda.current_stream(dev))     # after the allocations: whoever held the blocks is done
            self._deferred = (side, fork, plan, bufs)

    def _launch_deferred(self) -> None:
        side, fork, plan, bufs = self._deferred
        self._deferred = None
        tag = getattr(self.be, "tag", None)
        self._tag(None)                                         # per-block tables book the pack under "other"
        try:
            self._launch_deferred_inner(side, fork, plan, bufs)
        finally:
            if tag is not None:
                self.be.tag = tag

    def _launch_deferred_inner(self, side, fork, plan, bufs) -> None:
        if side is None:
            if plan is not None:
                self.be.pack_launch(plan)
            for b in bufs or ():
                b.zero_()
            return
        if plan is not None:
            self.be.pack_launch(plan, stream=side, after=fork)
        else:
            side.wait_event(fork)
        if bufs is not None:
            with torch.cuda.stream(side):
                for b in bufs:
                    b.zero_()
        self._fwd_side = side

    def _join_fwd_side(self) -> None:
        """the main stream waits for the forward-time side work (late pack, zero fills)"""
        if self._fwd_side is not None:
            torch.cuda.current_stream(self._fwd_side.device).wait_stream(self._fwd_side)
            self._fwd_side = None
        self._late = set()

    def _early_unpack(self) -> None:
        """OV_UNPACK (single GPU; data parallel has ``_flush_bucket`` at the same place): the weight gradients
        accumulated so far go to parameter layout on the side stream, in stream order behind the kernels that produced
        them; the unpack at the end of backward only handles the remaining (small, full-resolution) layers."""
        if not (self._ov & OV_UNPACK) or self.bucket_hook is not None or not self._unpack_list:
            return
        items, self._unpack_list = self._unpack_list, []
        side = self._side
        if side is None:
            self.be.unpack_many(items)
            return
        self.be.unpack_many(items, stream=side)     # the side stream first waits for the main stream's position
        self._side_keep.append(items)

    def _join_side(self) -> None:
        if self._side is not None:
            torch.cuda.current_stream(self._side.device).wait_stream(self._side)
            self._side = None
        self._side_keep = []

    def _flush_bucket(self, first_name: str) -> None:
        """Data parallel (SURVEY.md 8e): every gradient from parameter ``first_name`` to the end of the state_dict
        (the deepest encoder block, the whole decoder and the head = what backward has finished so far) is final ->
        unpack those weight gradients now and let the caller start their all-reduce under the rest of backward."""
        if self.bucket_hook is None:
            return
        self._join_side()
        self.be.unpack_many(self._unpack_list)
        self._unpack_list = []
        self.bucket_hook(self._flat, self._goff[first_name])

    def _finish_backward(self) -> None:
        self._join_side()
        self._tag(None)
        self.be.unpack_many(self._unpack_list)
        self._unpack_list = []
        self._packs = {}
        self._pre_bwd = None

    def _tag(self, wname: Optional[str]) -> None:
        """instrumentation hook: a profiling wrapper around the backend (bench.py) learns which network block
        (``in_tr``, ``down_tr32`` ... -- the first component of the parameter name) the next launches belong to"""
        if hasattr(self.be, "tag"):
            self.be.tag = wname.split(".")[0] if wname else "other"

    # ---------------------------------------------------------------- forward primitives
    def conv_raw(self, kind: int, wname: str, bname: Optional[str], x: Tensor, y: Tensor,
                 stats: Optional[Tensor] = None) -> None:
        w = self.P[wname]
        if wname in self._late:
            if self._deferred is not None:
                self._launch_deferred()
            self._join_fwd_side()
        wpk = self._packs.get((wname, "fwd"))
        if wpk is None:
            wpk = self.be.pack_weight(w, kind, "fwd", self.T, self.dims, vox=y.numel() // (y.shape[0] * y.shape[-1]))
        bias = self.P[bname] if bname is not None else None
        self.be.conv(kind, self.dims, x, wpk, bias, y, stats, None)
        if self._deferred is not None:
            self._launch_deferred()                    # behind the first convolution of the pass

    def conv_gn(self, kind: int, wname: str, bname: Optional[str], gname: str, x: Tensor,
                out_sp: Sequence[int], cout: int, drop: bool = True) -> Layer:
        """conv + stats + finalize.  The activation itself is produced later by ``apply``.  ``drop=False``: a layer
        without Dropout (it takes no mask from the pass's list)."""
        L = Layer(kind, wname, bname, gname, x=x)
        self._tag(wname)
        n = x.shape[0]
        L.y = self.new(x, out_sp, cout)
        stats = self.zeros((n, cout, 2), torch.float64, x.device)
        self.conv_raw(kind, wname, bname, x, L.y, stats)
        L.scale = self._next_mask() if drop else None
        vox = 1
        for s in out_sp:
            vox *= s
        if cout <= 512:
            # kernels derive the coefficients from the statistics themselves: no finalize launch
            # (wider layers -- init_features >= 64 -- take the finalize/apply form: any channel count)
            L.gn = (stats, self.P[gname + ".weight"], self.P[gname + ".bias"], L.scale, vox,
                    self.spec.groups or cout, GN_EPS)
            if self.spec.act != ACT_RELU:
                L.gn += (self.spec.act,)
        else:
            if self.spec != VNET:
                raise ValueError(f"the InstanceNorm / LeakyReLU layers take at most 512 channels, got {cout}")
            L.coef = torch.empty((n, cout, 2), dtype=torch.float32, device=x.device)
            L.mr = torch.empty((n, GROUPS, 2), dtype=torch.float32, device=x.device)
            self.be.gn_finalize(stats, self.P[gname + ".weight"], self.P[gname + ".bias"], L.scale, vox,
                                GROUPS, GN_EPS, L.coef, L.mr)
        self.layers.append(L)
        return L

    def stem_gn_ok(self, x: Tensor, f: int) -> bool:
        """can the input block run fused (``stem_block``)?  bf16 storage, one image channel, 16 features, and a backend
        with the fused kernels (the emulated CPU backend and the fp32 parity mode keep the per-branch calls)"""
        ok = getattr(self.be, "stem_gn_ok", None)
        return (ok is not None and self.spec.act == ACT_RELU and self.spec.groups == GROUPS and self.T == torch.bfloat16
                and f == 16 and ok(x, f, self.dims))

    def stem_block(self, x: Tensor, sp0, f: int, out: Tensor, drop: bool) -> Tuple[Layer, Layer]:
        """InputTransition (VNet3d.py:34-43, ResNet3d.py:24-41): relu(bn1(conv1(x))) + relu(bn1(conv2(x))) with the
        dropout of each branch, in two launches -- the statistics of both branches, then the normalised sum written
        into ``out``.  The raw stem outputs are never stored: both passes recompute them from the image."""
        n = x.shape[0]
        La = Layer(K3, "in_tr.conv1.weight", "in_tr.conv1.bias", "in_tr.bn1", x=x)
        Lb = Layer(K1, "in_tr.conv2.weight", "in_tr.conv2.bias", "in_tr.bn1", x=x)
        self._tag(La.wname)
        for L in (La, Lb):
            L.wpk = self._packs.get((L.wname, "fwd"))
            if L.wpk is None:
                L.wpk = self.be.pack_weight(self.P[L.wname], L.kind, "fwd", self.T, self.dims,
                                            vox=sp0[0] * sp0[1] * sp0[2])
        stats = [self.zeros((n, f, 2), torch.float64, x.device) for _ in range(2)]
        P = self.P
        self.be.stem_gn_stats(x, La.wpk, P[La.bname], Lb.wpk, P[Lb.bname], stats[0], stats[1])
        if self._deferred is not None:
            self._launch_deferred()                    # behind the first launch of the pass
        vox = sp0[0] * sp0[1] * sp0[2]
        for L, st in zip((La, Lb), stats):             # the masks in branch order, as conv_gn draws them
            L.scale = self._next_mask() if drop else None
            L.gn = (st, P[L.gname + ".weight"], P[L.gname + ".bias"], L.scale, vox, GROUPS, GN_EPS)
            self.layers.append(L)
        self._tag(La.wname)
        self.be.stem_gn_apply(x, La.wpk, P[La.bname], Lb.wpk, P[Lb.bname], La.gn, Lb.gn, out)
        return La, Lb

    def stem_block_backward(self, La: Layer, Lb: Layer, g: Tensor) -> None:
        """Backward of ``stem_block`` (no data gradient): the GroupNorm-backward sums of both branches in one pass
        over g, then dy of both branches formed on chip and consumed there by both stem weight gradients (+ d gamma,
        d beta and both bias gradients) in a second one."""
        be, P, dev = self.be, self.P, g.device
        self._tag(La.wname)
        n, f = g.shape[0], g.shape[-1]
        sums = [self.zeros((n, f, 3), torch.float64, dev) for _ in range(2)]
        be.stem_gn_bwd_sums(La.x, La.wpk, P[La.bname], Lb.wpk, P[Lb.bname], La.gn, Lb.gn, g, sums[0], sums[1])
        dwa = self.zeros((_taps(La.kind, self.dims), 1, f), torch.float32, dev)
        dwb = self.zeros((1, 1, f), torch.float32, dev)
        gv = self._grad_view
        be.stem_gn_bwd(La.x, La.wpk, P[La.bname], Lb.wpk, P[Lb.bname], La.gn, Lb.gn, g, sums[0], sums[1], dwa, dwb,
                       gv(La.gname + ".weight"), gv(La.gname + ".bias"), gv(La.bname), gv(Lb.bname))
        self._unpack_list.append((dwa, gv(La.wname)))
        self._unpack_list.append((dwb, gv(Lb.wname)))

    def up_gn_ok(self, x: Tensor, wname: str, co: int) -> bool:
        """can this transposed-conv layer run fused (``up_block``)?  bf16 storage, 3-D, 32 -> 16 channels at the shapes of
        the pointwise mma.sync kernel, and a backend with the fused kernels (the emulated CPU backend and the fp32
        parity mode keep the per-layer calls)"""
        ok = getattr(self.be, "up_gn_ok", None)
        if ok is None or self.T != torch.bfloat16 or self.dims != 3 or self.spec.act != ACT_RELU \
                or self.spec.groups != GROUPS:
            return False
        return ok(x, self._packs.get((wname, "fwd")), co, self.dims)

    def up_block(self, name: str, x: Tensor, sp, co: int, out: Tensor) -> Layer:
        """UpTransition's up_conv -> bn -> Dropout -> ReLU (VNet3d.py:62-72) in two launches -- the statistics, then the
        normalised activation written into ``out`` (the left half of the skip concat).  The raw transposed-conv output
        is never stored: both passes recompute it from ``x``."""
        L = Layer(UP, name + ".up_conv.weight", name + ".up_conv.bias", name + ".bn", x=x)
        self._tag(L.wname)
        if L.wname in self._late:
            if self._deferred is not None:
                self._launch_deferred()
            self._join_fwd_side()
        L.wpk = self._packs[(L.wname, "fwd")]
        n = x.shape[0]
        stats = self.zeros((n, co, 2), torch.float64, x.device)
        P = self.P
        self.be.up_gn_stats(x, L.wpk, P[L.bname], stats)
        L.scale = self._next_mask()
        L.gn = (stats, P[L.gname + ".weight"], P[L.gname + ".bias"], L.scale, sp[0] * sp[1] * sp[2], GROUPS, GN_EPS)
        self.layers.append(L)
        self.be.up_gn_apply(x, L.wpk, P[L.bname], L.gn, out)
        return L

    def up_block_backward(self, L: Layer, g: Tensor) -> Tensor:
        """Backward of ``up_block``: the GroupNorm-backward sums in one pass over g, then dy formed on chip and consumed
        there by the weight gradient and the data gradient (+ d gamma, d beta and the bias gradient) in a second one.
        Returns the gradient w.r.t. the layer input."""
        be, dev = self.be, g.device
        self._tag(L.wname)
        n, co = g.shape[0], g.shape[-1]
        sums = self.zeros((n, co, 3), torch.float64, dev)
        bias = self.P[L.bname]
        be.up_gn_bwd_sums(L.x, L.wpk, bias, L.gn, g, sums)
        dwp = self.zeros((_taps(UP, self.dims), co, L.x.shape[-1]), torch.float32, dev)
        dx = torch.empty(L.x.shape, dtype=self.T, device=dev)
        gv = self._grad_view
        be.up_gn_bwd(L.x, L.wpk, bias, L.gn, g, sums, dwp, dx, gv(L.gname + ".weight"), gv(L.gname + ".bias"),
                     gv(L.bname))
        self._unpack_list.append((dwp, gv(L.wname)))
        return dx

    def head(self, wname: str, bname: str, x: Tensor, sp0, ncls: int) -> Tuple[Layer, Tensor, Optional[Tensor]]:
        """OutputTransition3d / UNet head: 1x1 conv to the classes + sigmoid/softmax (VNet3d.py:90-99).
        Inference form (``mask_threshold`` set; predict, model/modelVNet.py:655-676): the uint8 mask directly."""
        self._tag(wname)
        if self._deferred is not None:
            self._launch_deferred()
        self._join_fwd_side()                      # the last forward op: nothing of this pass stays un-joined
        if self.mask_threshold is not None:
            mask = torch.empty((x.shape[0],) + tuple(sp0), dtype=torch.uint8, device=x.device)
            if not self.be.head_mask(x, self.P[wname], self.P[bname], mask, float(self.mask_threshold)):
                logits = self.new(x, sp0, ncls, dtype=torch.float32)
                self.conv_raw(K1, wname, bname, x, logits)
                self.be.mask_logits(logits, float(self.mask_threshold), mask)
            return None, mask, None
        logits = self.new(x, sp0, ncls, dtype=torch.float32)
        probs = torch.empty_like(logits) if self.want_probs else None
        Lh = Layer(K1, wname, bname, None, x=x, y=logits)
        if not self.be.head_fwd(x, self.P[wname], self.P[bname], logits, probs):
            self.conv_raw(K1, wname, bname, x, logits)
            if probs is not None:
                self.be.head_probs(logits, probs)
        return Lh, logits, probs

    def head_backward(self, Lh: Layer, g_logits: Tensor) -> Tensor:
        self._tag(Lh.wname)
        dx = torch.empty(Lh.x.shape, dtype=self.T, device=g_logits.device)
        if self.be.head_bwd(Lh.x, g_logits, self.P[Lh.wname], dx, self._grad_view(Lh.wname), self._grad_view(Lh.bname)):
            return dx
        return self.bwd_layer(Lh, g_logits, True, dx_out=dx)

    def act(self, L: Layer, out: Tensor, L2: Optional[Layer] = None, res: Optional[Tensor] = None) -> Tensor:
        self._tag(L.wname)
        if L.gn is not None:
            self.be.apply_gn(L.y, L.gn, L2.y if L2 is not None else None, L2.gn if L2 is not None else None, res, out)
        else:
            self.be.apply(L.y, L.coef, L2.y if L2 is not None else None, L2.coef if L2 is not None else None, res, out)
        return out

    # ---------------------------------------------------------------- backward primitives
    def _grad_view(self, name: str) -> Tensor:
        return self.grads[name]

    def bwd_layer(self, L: Layer, g_act: Tensor, need_dx: bool, dx_out: Optional[Tensor] = None,
                  dx_addend: Optional[Tensor] = None, prev: Optional[Layer] = None,
                  side_wgrad: bool = False) -> Optional[Tensor]:
        """Backward of one conv(+GN/drop/ReLU) application.  ``g_act`` is the gradient w.r.t.
        the layer's activation output (or w.r.t. the raw conv output when the layer has no
        GroupNorm).  Returns the gradient w.r.t. the layer input (written to ``dx_out``).
        ``prev``: the GroupNorm layer whose activation IS this layer's input and whose complete activation gradient
        this call produces (data gradient + ``dx_addend``): where the kernel can, the first pass of ``prev``'s
        GroupNorm backward (the sums over g and its raw output) is folded into the data-gradient epilogue."""
        be = self.be
        self._tag(L.wname)
        n, cout = L.y.shape[0], L.y.shape[-1]
        dev = L.y.device
        vox = L.y.numel() // (n * cout)
        if L.gname is not None and L.gn is not None:
            dy = torch.empty(L.y.shape, dtype=self.T, device=dev)
            dgam, dbet = self._grad_view(L.gname + ".weight"), self._grad_view(L.gname + ".bias")
            dbia = self._grad_view(L.bname) if L.bname is not None else None
            fused = getattr(be, "gn_bwd_fused_ok", None)
            if L.pre_sums is not None:
                # the conv that produced g_act has already accumulated sum g*m and sum g*m*y in its epilogue
                be.gn_bwd_apply_gn(g_act, L.y, L.gn, L.pre_sums, dy, dgam, dbet, dbia, sum_y_from_stats=True)
                L.pre_sums = None
            elif fused is not None and fused(g_act, L.y, dy):
                # small levels: reduce -> grid barrier -> apply in one launch (sums + one zeroed barrier word)
                buf = self.zeros((n * cout * 3 + 2,), torch.float64, dev)
                be.gn_bwd_fused_gn(g_act, L.y, L.gn, buf[:n * cout * 3].view(n, cout, 3), buf[n * cout * 3:], dy,
                                   dgam, dbet, dbia)
            else:
                sums = self.zeros((n, cout, 3), torch.float64, dev)
                be.gn_bwd_reduce_gn(g_act, L.y, L.gn, sums)
                be.gn_bwd_apply_gn(g_act, L.y, L.gn, sums, dy, dgam, dbet, dbia)
        elif L.gname is not None:
            sums = self.zeros((n, cout, 3), torch.float64, dev)
            be.gn_bwd_reduce(g_act, L.y, L.coef, sums)
            coef3 = torch.empty((n, cout, 3), dtype=torch.float32, device=dev)
            be.gn_bwd_finalize(sums, L.mr, self.P[L.gname + ".weight"], L.scale, vox, GROUPS, coef3,
                               self._grad_view(L.gname + ".weight"), self._grad_view(L.gname + ".bias"),
                               self._grad_view(L.bname) if L.bname is not None else None)
            dy = torch.empty(L.y.shape, dtype=self.T, device=dev)
            be.gn_bwd_apply(g_act, L.y, L.coef, coef3, dy)
        else:
            dy = g_act
            if L.bname is not None:
                be.colsum(dy, self._grad_view(L.bname))
        w = self.P[L.wname]
        if not self._data_only:
            self._wgrad(L, dy, side=need_dx or side_wgrad)
        if not need_dx:
            return None
        wd = self._packs.get((L.wname, "dgrad"))
        if wd is None:
            wd = be.pack_weight(w, L.kind, "dgrad", self.T, self.dims,
                                vox=L.x.numel() // (L.x.shape[0] * L.x.shape[-1]))
        dkind = {K3: K3, K1: K1, DOWN: UP, UP: DOWN}[L.kind]
        if dx_out is None:
            dx_out = torch.empty(L.x.shape, dtype=self.T, device=dev)
        ok = getattr(be, "conv_bwdstats_ok", None)
        # (the fused backward-sums epilogue has the ReLU tail only: a LeakyReLU layer takes the two-pass form)
        if (prev is not None and prev.gn is not None and prev.gname is not None and ok is not None
                and len(prev.gn) == 7 and prev.y.shape == dx_out.shape
                and ok(dkind, self.dims, dy, wd, dx_out, dx_addend, prev.y)):
            self._tag(prev.wname)
            prev.pre_sums = self.zeros((prev.y.shape[0], prev.y.shape[-1], 3), torch.float64, dev)
            be.conv_bwdstats(dkind, self.dims, dy, wd, dx_out, dx_addend, prev.y, prev.gn, prev.pre_sums)
        else:
            be.conv(dkind, self.dims, dy, wd, None, dx_out, None, dx_addend)
        return dx_out

    def _wgrad(self, L: Layer, dy: Tensor, side: bool) -> None:
        """the weight gradient of ``bwd_layer``, queued for the final unpack"""
        be, dev = self.be, dy.device
        taps = _taps(L.kind, self.dims)
        cin, cout = L.x.shape[-1], L.y.shape[-1]
        if L.kind == UP:
            dwp = self.zeros((taps, cout, cin), torch.float32, dev)
            wg = (DOWN, self.dims, dy, L.x, dwp)             # a = fine side (dy), b = coarse side (x)
        else:
            dwp = self.zeros((taps, cin, cout), torch.float32, dev)
            wg = (L.kind, self.dims, L.x, dy, dwp)
        # without a data gradient there is nothing to overlap with, unless the caller has more work for the main
        # stream (``side_wgrad``: the other branch of the input block)
        st = _side_stream(dev) if side else None
        if st is not None:
            # dW only feeds the final unpack: run it beside the dgrad -> next-layer chain
            st.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(st):
                be.wgrad(*wg)
            self._side = st
            self._side_keep.append(wg)
        else:
            be.wgrad(*wg)
        self._unpack_list.append((dwp, self._grad_view(L.wname)))

    def alloc_grads(self, device) -> Tensor:
        """One flat fp32 bucket; ``self.grads`` are views in state_dict order (the bucket is
        what the data-parallel all-reduce sums, SURVEY.md section 8e)."""
        total = sum(p.numel() for p in self.P.values())
        if self._pre_bwd is not None and self._pre_bwd[0].numel() == total:
            flat = self._pre_bwd[0]                       # zeroed on the side stream during forward (OV_ZERO)
        else:
            flat = torch.zeros(total, dtype=torch.float32, device=device)
        off = 0
        self.grads, self._goff, self._flat = {}, {}, flat
        for name, p in self.P.items():
            self.grads[name] = flat[off:off + p.numel()].view(p.shape)
            self._goff[name] = off
            off += p.numel()
        return flat

    # ================================================================== VNet3d
    def _out_views(self, logits: Tensor, probs: Optional[Tensor]):
        """(N,D,H,W,C) channels-last buffers -> the NCDHW / NCHW-shaped (channels-last-strided) tensors of the
        nn.Module contract; a uint8 inference mask (N,D,H,W) loses the unit depth of the 2-D nets."""
        if logits.dtype == torch.uint8:
            return (logits if self.dims == 3 else logits[:, 0]), None
        if self.dims == 3:
            return logits.permute(0, 4, 1, 2, 3), (probs.permute(0, 4, 1, 2, 3) if probs is not None else None)
        return logits[:, 0].permute(0, 3, 1, 2), (probs[:, 0].permute(0, 3, 1, 2) if probs is not None else None)

    def vnet_forward(self, P: Dict[str, Tensor], x: Tensor, masks: Optional[List[Tensor]],
                     need_grad: bool, spec: VNetSpec = VNET) -> Tuple[Tensor, Tensor]:
        """VNet3d.forward (reference networks/VNet3d.py:129-158) and its 2-D twin VNet2d.forward
        (networks/VNet2d.py:129-158; 2-D tensors run with a unit depth).  ``x``: (N,Cin,[D,]H,W) fp32.
        Returns channels-last-strided (N,ncls,[D,]H,W) fp32 logits and probs.  ``spec=REGISTRATION``: the network of
        VNet3dRegistration up to its displacement field (networks/VNet3dregistration.py:174-203)."""
        self.P, self.masks, self._mi, self.layers, self.need_grad = P, masks, 0, [], need_grad
        self.spec = spec
        oc, ob = spec.op_conv, spec.op_bn
        downs = tuple(zip(("down_tr32", "down_tr64", "down_tr128", "down_tr256"), spec.down_ops))
        ups = tuple(zip(("up_tr256", "up_tr128", "up_tr64", "up_tr32"), spec.up_ops))
        sv = self.saved = {}
        dims = self.dims
        n, cin = x.shape[0], x.shape[1]
        self._begin_pass(n, x.device, backward=False)
        if dims == 3:
            sp0 = tuple(x.shape[2:])
            xin = x.permute(0, 2, 3, 4, 1)
        else:
            sp0 = (1,) + tuple(x.shape[2:])
            xin = x.permute(0, 2, 3, 1).unsqueeze(1)
        if cin != 1:
            xin = xin.contiguous()
        f = P["in_tr.conv1.weight"].shape[0]
        sps = [sp0]
        for _ in range(4):
            s_ = sps[-1]
            sps.append((s_[0] // 2 if dims == 3 else 1, s_[1] // 2, s_[2] // 2))
        ch = [f, 2 * f, 4 * f, 8 * f, 16 * f]
        # skip-concat buffers of the four UpTransitions: [up | skip], VNet3d.py:74
        cats = [self.new(x, sps[i], 2 * ch[i]) for i in range(4)]
        skips = [cats[i][..., ch[i]:] for i in range(4)]

        vox = [sp[0] * sp[1] * sp[2] for sp in sps]
        specs = [("in_tr.conv1.weight", K3, vox[0], vox[0], False), ("in_tr.conv2.weight", K1, vox[0], vox[0], False)]
        for i, (name, nops) in enumerate(downs):
            specs.append((name + ".down_conv.weight", DOWN, vox[i + 1], vox[i], True))
            specs += [(f"{name}.ops.{j}.{oc}.weight", K3, vox[i + 1], vox[i + 1], True) for j in range(nops)]
        for i, (name, nops) in zip((3, 2, 1, 0), ups):
            specs.append((name + ".up_conv.weight", UP, vox[i], vox[i + 1], True))
            specs.append((name + ".conv.weight", K1, vox[i], vox[i], True))
            specs += [(f"{name}.ops.{j}.{oc}.weight", K3, vox[i], vox[i], True) for j in range(nops)]
        self._batch, self._ov = n, overlap_mask("vnet", dims)
        self._prepack(specs, need_grad, n_early=5)         # in_tr (2) + down_tr32 (down conv + 2 ops)

        # ---- InputTransition3d (VNet3d.py:34-43): one bn1 serves both branches
        if self.stem_gn_ok(xin, f):
            La, Lb = self.stem_block(xin, sp0, f, skips[0], drop=True)
            out = skips[0]
        else:
            ib = "in_tr." + spec.in_bn
            La = self.conv_gn(K3, "in_tr.conv1.weight", "in_tr.conv1.bias", ib, xin, sp0, f)
            Lb = self.conv_gn(K1, "in_tr.conv2.weight", "in_tr.conv2.bias", ib, xin, sp0, f)
            out = self.act(La, skips[0], L2=Lb)
        sv["in_tr"] = (La, Lb)

        # ---- DownTransition3d x4 (VNet3d.py:55-59)
        for i, (name, nops) in enumerate(downs):
            co, sp = ch[i + 1], sps[i + 1]
            Ld = self.conv_gn(DOWN, name + ".down_conv.weight", name + ".down_conv.bias", f"{name}.{spec.down_bn}",
                              out, sp, co)
            down = self.act(Ld, self.new(x, sp, co))
            h, ops = down, []
            for j in range(nops):
                Lo = self.conv_gn(K3, f"{name}.ops.{j}.{oc}.weight", f"{name}.ops.{j}.{oc}.bias",
                                  f"{name}.ops.{j}.{ob}", h, sp, co)
                ops.append(Lo)
                last = j == nops - 1
                if last:
                    dst = skips[i + 1] if i + 1 < 4 else self.new(x, sp, co)
                    h = self.act(Lo, dst, res=down)                     # torch.add(out, down), VNet3d.py:58
                else:
                    h = self.act(Lo, self.new(x, sp, co))
            sv[name] = (Ld, ops)
            out = h

        # ---- UpTransition3d x4 (VNet3d.py:72-80)
        for i, (name, nops) in zip((3, 2, 1, 0), ups):
            co, sp = ch[i], sps[i]
            if name == "up_tr32" and self.up_gn_ok(out, name + ".up_conv.weight", co):
                Lu = self.up_block(name, out, sp, co, cats[i][..., :co])
            else:
                Lu = self.conv_gn(UP, name + ".up_conv.weight", name + ".up_conv.bias", name + ".bn", out, sp, co)
                self.act(Lu, cats[i][..., :co])                          # left half of the concat
            Lc = self.conv_gn(K1, name + ".conv.weight", name + ".conv.bias", name + ".bn", cats[i], sp, co)
            xcat = self.act(Lc, self.new(x, sp, co))
            h, ops = xcat, []
            for j in range(nops):
                Lo = self.conv_gn(K3, f"{name}.ops.{j}.{oc}.weight", f"{name}.ops.{j}.{oc}.bias",
                                  f"{name}.ops.{j}.{ob}", h, sp, co)
                ops.append(Lo)
                last = j == nops - 1
                h = self.act(Lo, self.new(x, sp, co), res=xcat if last else None)   # VNet3d.py:79
            sv[name] = (Lu, Lc, ops)
            out = h

        # ---- OutputTransition3d (VNet3d.py:90-99)
        ncls = P["out_tr.conv.weight"].shape[0]
        Lh, logits, probs = self.head("out_tr.conv.weight", "out_tr.conv.bias", out, sp0, ncls)
        sv["head"] = Lh
        return self._out_views(logits, probs)

    vnet3d_forward = vnet_forward

    def vnet_backward(self, g_logits: Tensor) -> Tensor:
        """Gradients of all 128 parameters given d loss / d logits ((N,D,H,W,ncls) fp32,
        channels-last).  Returns the flat fp32 bucket; ``self.grads`` holds the views."""
        sv = self.saved
        flat = self.alloc_grads(g_logits.device)
        self._begin_pass(g_logits.shape[0], g_logits.device, backward=True)
        g = self.head_backward(sv["head"], g_logits)
        gskip: List[Optional[Tensor]] = [None] * 4
        for i, name in zip((0, 1, 2, 3), ["up_tr32", "up_tr64", "up_tr128", "up_tr256"]):
            Lu, Lc, ops = sv[name]
            g_out = g                                    # d/d(out) ; out = ops(xcat) + xcat
            gh = g_out
            for j in reversed(range(len(ops))):
                gh = self.bwd_layer(ops[j], gh, True, dx_addend=g_out if j == 0 else None,
                                    prev=ops[j - 1] if j > 0 else Lc)
            gcat = self.bwd_layer(Lc, gh, True)          # (N,..,2*co)
            co = Lc.y.shape[-1]
            gskip[i] = gcat[..., co:]
            if Lu.wpk is not None:
                g = self.up_block_backward(Lu, gcat[..., :co])
            else:
                g = self.bwd_layer(Lu, gcat[..., :co], True)
        for i, name in zip((3, 2, 1, 0), ["down_tr256", "down_tr128", "down_tr64", "down_tr32"]):
            Ld, ops = sv[name]
            g_out = g
            gh = g_out
            for j in reversed(range(len(ops))):
                gh = self.bwd_layer(ops[j], gh, True, dx_addend=g_out if j == 0 else None,
                                    prev=ops[j - 1] if j > 0 else Ld)
            g = self.bwd_layer(Ld, gh, True, dx_addend=gskip[i])
            if i == 3:
                self._flush_bucket("down_tr256.down_conv.weight")
                self._early_unpack()
        La, Lb = sv["in_tr"]
        if La.wpk is not None:
            self.stem_block_backward(La, Lb, g)
        else:
            self.bwd_layer(La, g, False, side_wgrad=bool(self._ov & OV_TAIL))
            self.bwd_layer(Lb, g, False)
        self._finish_backward()
        return flat

    vnet3d_backward = vnet_backward

    # ================================================================== ResNet3d / ResNet2d
    def resnet_forward(self, P: Dict[str, Tensor], x: Tensor, masks: Optional[List[Tensor]],
                       need_grad: bool) -> Tensor:
        """ResNet3d.forward / ResNet2d.forward (reference networks/ResNet3d.py:98-118, ResNet2d.py:99-119): the VNet
        encoder with Dropout only in the four DownTransitions, then GlobalAveragePooling -> Linear -> ReLU -> Linear.
        ``do1`` (ResNet3d.py:51-55) drops ``down`` in place, so the residual adds the dropped tensor too: the same
        algebra as the VNet down block.  ``x``: (N,Cin,[D,]H,W) fp32.  Returns (N, numclass) fp32 logits."""
        self.P, self.masks, self._mi, self.layers, self.need_grad = P, masks, 0, [], need_grad
        sv = self.saved = {}
        dims = self.dims
        n, cin = x.shape[0], x.shape[1]
        self._begin_pass(n, x.device, backward=False)
        if dims == 3:
            sp0 = tuple(x.shape[2:])
            xin = x.permute(0, 2, 3, 4, 1)
        else:
            sp0 = (1,) + tuple(x.shape[2:])
            xin = x.permute(0, 2, 3, 1).unsqueeze(1)
        if cin != 1:
            xin = xin.contiguous()
        f = P["in_tr.conv1.weight"].shape[0]
        sps = [sp0]
        for _ in range(4):
            s_ = sps[-1]
            sps.append((s_[0] // 2 if dims == 3 else 1, s_[1] // 2, s_[2] // 2))
        ch = [f, 2 * f, 4 * f, 8 * f, 16 * f]
        vox = [sp[0] * sp[1] * sp[2] for sp in sps]
        nconvs = (("down_tr32", 2), ("down_tr64", 3), ("down_tr128", 3), ("down_tr256", 3))
        specs = [("in_tr.conv1.weight", K3, vox[0], vox[0], False), ("in_tr.conv2.weight", K1, vox[0], vox[0], False)]
        for i, (name, nops) in enumerate(nconvs):
            specs.append((name + ".down_conv.weight", DOWN, vox[i + 1], vox[i], True))
            specs += [(f"{name}.ops.{j}.conv1.weight", K3, vox[i + 1], vox[i + 1], True) for j in range(nops)]
        self._batch, self._ov = n, overlap_mask("resnet", dims)
        self._prepack(specs, need_grad, n_early=5)         # in_tr (2) + down_tr32 (down conv + 2 ops)

        # ---- InputTransition3d (ResNet3d.py:24-41): one bn1 for both branches, no dropout
        if self.stem_gn_ok(xin, f):
            out = self.new(x, sp0, f)
            La, Lb = self.stem_block(xin, sp0, f, out, drop=False)
        else:
            La = self.conv_gn(K3, "in_tr.conv1.weight", "in_tr.conv1.bias", "in_tr.bn1", xin, sp0, f, drop=False)
            Lb = self.conv_gn(K1, "in_tr.conv2.weight", "in_tr.conv2.bias", "in_tr.bn1", xin, sp0, f, drop=False)
            out = self.act(La, self.new(x, sp0, f), L2=Lb)
        sv["in_tr"] = (La, Lb)

        # ---- DownTransition3d x4 (ResNet3d.py:44-58): the LUConv stacks have no dropout
        for i, (name, nops) in enumerate(nconvs):
            co, sp = ch[i + 1], sps[i + 1]
            Ld = self.conv_gn(DOWN, name + ".down_conv.weight", name + ".down_conv.bias", name + ".bn1", out, sp, co)
            down = self.act(Ld, self.new(x, sp, co))
            h, ops = down, []
            for j in range(nops):
                Lo = self.conv_gn(K3, f"{name}.ops.{j}.conv1.weight", f"{name}.ops.{j}.conv1.bias",
                                  f"{name}.ops.{j}.bn1", h, sp, co, drop=False)
                ops.append(Lo)
                h = self.act(Lo, self.new(x, sp, co), res=down if j == nops - 1 else None)   # ResNet3d.py:57
            sv[name] = (Ld, ops)
            out = h

        # ---- GlobalAveragePooling + fc_layers (ResNet3d.py:61-69,93-96)
        self._tag("fc_layers")
        if self._deferred is not None:
            self._launch_deferred()
        self._join_fwd_side()                      # the last forward op: nothing of this pass stays un-joined
        w1, w2 = P["fc_layers.0.weight"], P["fc_layers.2.weight"]
        pooled = torch.empty((n, out.shape[-1]), dtype=torch.float32, device=x.device)
        hidden = torch.empty((n, w1.shape[0]), dtype=torch.float32, device=x.device)
        logits = torch.empty((n, w2.shape[0]), dtype=torch.float32, device=x.device)
        self.be.cls_head_fwd(out, w1, P["fc_layers.0.bias"], w2, P["fc_layers.2.bias"], pooled, hidden, logits)
        sv["head"] = (out, pooled, hidden)
        return logits

    def resnet_backward(self, g_logits: Tensor, stages: Optional[Sequence[str]] = None):
        """Gradients of all 70 parameters given d loss / d logits ((N, numclass) fp32, contiguous).  Returns the flat
        fp32 bucket; ``self.grads`` holds the views.

        ``stages`` (Grad-CAM): names from ``RESNET_STAGES``.  Then only data gradients are computed -- no weight-gradient
        convolution runs, the GroupNorm, bias and head parameter gradients land in a scratch bucket -- and the pass stops
        after the earliest stage asked for.  Returns {stage: (output, d loss / d output)}, channels-last in the engine's
        dtype; the output of ``in_tr`` is the input of ``down_tr32.down_conv``, that of ``down_tr256`` the head input."""
        sv = self.saved
        dev = g_logits.device
        want = set(stages or ())
        self._data_only = stages is not None
        flat = self.alloc_grads(dev)
        n = g_logits.shape[0]
        self._begin_pass(n, dev, backward=True)
        out, pooled, hidden = sv["head"]
        self._tag("fc_layers")
        w1, w2 = self.P["fc_layers.0.weight"], self.P["fc_layers.2.weight"]
        g = torch.empty(out.shape, dtype=self.T, device=dev)
        work = torch.empty(n * (w1.shape[0] + w1.shape[1]), dtype=torch.float32, device=dev)
        gv = self._grad_view
        self.be.cls_head_bwd(g_logits, pooled, hidden, w1, w2, work, g, gv("fc_layers.0.weight"),
                             gv("fc_layers.0.bias"), gv("fc_layers.2.weight"), gv("fc_layers.2.bias"))
        found = {}
        for i, name in zip((3, 2, 1, 0), ["down_tr256", "down_tr128", "down_tr64", "down_tr32"]):
            Ld, ops = sv[name]
            if name in want:
                found[name] = (out, g)
                if len(found) == len(want):
                    break
            g_out = g                                    # d/d(out) ; out = ops(down) + down
            gh = g_out
            for j in reversed(range(len(ops))):
                gh = self.bwd_layer(ops[j], gh, True, dx_addend=g_out if j == 0 else None,
                                    prev=ops[j - 1] if j > 0 else Ld)
            g = self.bwd_layer(Ld, gh, True)
            out = Ld.x                                   # the previous stage's output
            if i == 3 and not self._data_only:
                self._flush_bucket("down_tr256.down_conv.weight")
                self._early_unpack()
        else:
            if "in_tr" in want:
                found["in_tr"] = (out, g)
            elif not self._data_only:
                La, Lb = sv["in_tr"]
                if La.wpk is not None:
                    self.stem_block_backward(La, Lb, g)
                else:
                    self.bwd_layer(La, g, False, side_wgrad=bool(self._ov & OV_TAIL))
                    self.bwd_layer(Lb, g, False)
        self._finish_backward()
        self._data_only = False
        return found if stages is not None else flat

    # ================================================================== UNet3d / UNet2d
    def unet_forward(self, P: Dict[str, Tensor], x: Tensor, masks: Optional[List[Tensor]],
                     need_grad: bool) -> Tuple[Tensor, Tensor]:
        """UNet3d.forward / UNet2d.forward (reference networks/Unet3d.py:36-62, Unet2d.py:36-62)."""
        self.P, self.masks, self._mi, self.layers, self.need_grad = P, masks, 0, [], need_grad
        sv = self.saved = {}
        dims = self.dims
        n, cin = x.shape[0], x.shape[1]
        self._begin_pass(n, x.device, backward=False)
        if dims == 3:
            sp0 = tuple(x.shape[2:])
            xin = x.permute(0, 2, 3, 4, 1)
        else:
            sp0 = (1,) + tuple(x.shape[2:])
            xin = x.permute(0, 2, 3, 1).unsqueeze(1)
        if cin != 1:
            xin = xin.contiguous()
        f = P["encoder1.enc1conv1.weight"].shape[0]
        ch = [f, 2 * f, 4 * f, 8 * f, 16 * f]
        sps = [sp0]
        for _ in range(4):
            s = sps[-1]
            sps.append((s[0] // 2 if dims == 3 else 1, s[1] // 2, s[2] // 2))
        cats = [self.new(x, sps[i], 2 * ch[i]) for i in range(4)]
        vox = [sp[0] * sp[1] * sp[2] for sp in sps]
        specs = []
        for i, (mod, name) in enumerate((("encoder1", "enc1"), ("encoder2", "enc2"), ("encoder3", "enc3"),
                                         ("encoder4", "enc4"), ("bottleneck", "bottleneck"))):
            specs.append((f"{mod}.{name}conv1.weight", K3, vox[i], vox[i], i > 0))
            specs.append((f"{mod}.{name}conv2.weight", K3, vox[i], vox[i], True))
        for i in (3, 2, 1, 0):
            specs.append((f"upconv{i + 1}.weight", UP, vox[i], vox[i + 1], True))
            specs.append((f"decoder{i + 1}.dec{i + 1}conv1.weight", K3, vox[i], vox[i], True))
            specs.append((f"decoder{i + 1}.dec{i + 1}conv2.weight", K3, vox[i], vox[i], True))
        self._batch, self._ov = n, overlap_mask("unet", dims)
        self._prepack(specs, need_grad, n_early=2)         # encoder1

        def block(mod: str, name: str, h: Tensor, sp, co: int, dst: Tensor):
            L1 = self.conv_gn(K3, f"{mod}.{name}conv1.weight", None, f"{mod}.{name}norm1", h, sp, co)
            a1 = self.act(L1, self.new(x, sp, co))
            L2 = self.conv_gn(K3, f"{mod}.{name}conv2.weight", None, f"{mod}.{name}norm2", a1, sp, co)
            a2 = self.act(L2, dst)
            sv[mod] = (L1, L2)
            return a2

        h = xin
        encs = []
        for i in range(4):
            e = block(f"encoder{i + 1}", f"enc{i + 1}", h, sps[i], ch[i], cats[i][..., ch[i]:])
            encs.append(e)
            h = self.new(x, sps[i + 1], ch[i])
            self.be.pool_fwd(e, h, dims)                                   # nn.MaxPool(2,2), Unet3d.py:18-24
            sv[f"pool{i + 1}"] = (e, h)
        h = block("bottleneck", "bottleneck", h, sps[4], ch[4], self.new(x, sps[4], ch[4]))
        for i in (3, 2, 1, 0):
            k = i + 1
            Lu = Layer(UP, f"upconv{k}.weight", f"upconv{k}.bias", None, x=h, y=cats[i][..., :ch[i]])
            self.conv_raw(UP, Lu.wname, Lu.bname, h, Lu.y)                 # no norm/act, Unet3d.py:44
            sv[f"upconv{k}"] = Lu
            h = block(f"decoder{k}", f"dec{k}", cats[i], sps[i], ch[i], self.new(x, sps[i], ch[i]))
        ncls = P["conv.weight"].shape[0]
        Lh, logits, probs = self.head("conv.weight", "conv.bias", h, sp0, ncls)
        sv["head"] = Lh
        return self._out_views(logits, probs)

    def unet_backward(self, g_logits: Tensor) -> Tensor:
        sv = self.saved
        flat = self.alloc_grads(g_logits.device)
        self._begin_pass(g_logits.shape[0], g_logits.device, backward=True)
        g = self.head_backward(sv["head"], g_logits)
        genc: List[Optional[Tensor]] = [None] * 4
        for i in (0, 1, 2, 3):
            k = i + 1
            L1, L2 = sv[f"decoder{k}"]
            g1 = self.bwd_layer(L2, g, True, prev=L1)
            gcat = self.bwd_layer(L1, g1, True)
            co = L2.y.shape[-1]
            genc[i] = gcat[..., co:]
            g = self.bwd_layer(sv[f"upconv{k}"], gcat[..., :co], True)
        L1, L2 = sv["bottleneck"]
        g = self.bwd_layer(L1, self.bwd_layer(L2, g, True, prev=L1), True)
        self._flush_bucket("bottleneck.bottleneckconv1.weight")
        self._early_unpack()
        for i in (3, 2, 1, 0):
            e, pooled = sv[f"pool{i + 1}"]
            ge = torch.empty(e.shape, dtype=self.T, device=e.device)
            self.be.pool_bwd(e, g, genc[i], ge, self.dims)               # + gradient from the skip concat
            L1, L2 = sv[f"encoder{i + 1}"]
            g1 = self.bwd_layer(L2, ge, True, prev=L1)
            g = self.bwd_layer(L1, g1, i > 0)
        self._finish_backward()
        return flat

    # ================================================================== UNet3dthin
    def unetthin_forward(self, P: Dict[str, Tensor], x: Tensor, masks: Optional[List[Tensor]],
                         need_grad: bool) -> Tuple[Tensor, Tensor]:
        """UNet3dthin.forward (reference networks/Unet3dthin.py:33-62): UNet3d's encoder, then four decoder blocks at
        the coarse resolution of their level, each followed by ``S = up2(block output) + encoder output``
        (nn.Upsample(2, trilinear) + torch.add, one kernel).  3-D only."""
        self.P, self.masks, self._mi, self.layers, self.need_grad = P, masks, 0, [], need_grad
        sv = self.saved = {}
        n, cin = x.shape[0], x.shape[1]
        self._begin_pass(n, x.device, backward=False)
        sp0 = tuple(x.shape[2:])
        xin = x.permute(0, 2, 3, 4, 1)
        if cin != 1:
            xin = xin.contiguous()
        f = P["encoder1.enc1conv1.weight"].shape[0]
        ch = [f, 2 * f, 4 * f, 8 * f, 16 * f]
        sps = [sp0]
        for _ in range(4):
            s = sps[-1]
            sps.append((s[0] // 2, s[1] // 2, s[2] // 2))
        vox = [sp[0] * sp[1] * sp[2] for sp in sps]
        specs = []
        for i, (mod, name) in enumerate((("encoder1", "enc1"), ("encoder2", "enc2"), ("encoder3", "enc3"),
                                         ("encoder4", "enc4"), ("bottleneck", "bottleneck"))):
            specs.append((f"{mod}.{name}conv1.weight", K3, vox[i], vox[i], i > 0))
            specs.append((f"{mod}.{name}conv2.weight", K3, vox[i], vox[i], True))
        for k in (4, 3, 2, 1):                              # decoder k runs at level k (the coarse side of its join)
            specs.append((f"decoder{k}.dec{k}conv1.weight", K3, vox[k], vox[k], True))
            specs.append((f"decoder{k}.dec{k}conv2.weight", K3, vox[k], vox[k], True))
        self._batch, self._ov = n, overlap_mask("unetthin", 3)
        self._prepack(specs, need_grad, n_early=2)         # encoder1

        def block(mod: str, name: str, h: Tensor, sp, co: int) -> Tensor:
            L1 = self.conv_gn(K3, f"{mod}.{name}conv1.weight", None, f"{mod}.{name}norm1", h, sp, co)
            a1 = self.act(L1, self.new(x, sp, co))
            L2 = self.conv_gn(K3, f"{mod}.{name}conv2.weight", None, f"{mod}.{name}norm2", a1, sp, co)
            a2 = self.act(L2, self.new(x, sp, co))
            sv[mod] = (L1, L2)
            return a2

        h = xin
        encs = []
        for i in range(4):
            e = block(f"encoder{i + 1}", f"enc{i + 1}", h, sps[i], ch[i])
            encs.append(e)
            h = self.new(x, sps[i + 1], ch[i])
            self.be.pool_fwd(e, h, 3)                                      # nn.MaxPool3d(2, 2), Unet3dthin.py:18-24
            sv[f"pool{i + 1}"] = (e, h)
        h = block("bottleneck", "bottleneck", h, sps[4], ch[4])
        for k in (4, 3, 2, 1):
            d = block(f"decoder{k}", f"dec{k}", h, sps[k], ch[k - 1])
            self._tag(f"decoder{k}")
            h = self.new(x, sps[k - 1], ch[k - 1])
            self.be.upsample_add(d, encs[k - 1], h)                       # Unet3dthin.py:41-42 (47, 51, 54)
        ncls = P["conv.weight"].shape[0]
        Lh, logits, probs = self.head("conv.weight", "conv.bias", h, sp0, ncls)
        sv["head"] = Lh
        return self._out_views(logits, probs)

    def unetthin_backward(self, g_logits: Tensor) -> Tensor:
        """Gradients of all 56 parameters given d loss / d logits.  The gradient of each join ``S_k`` goes twice: through
        up2^T into decoder k, and unchanged into the skip, where it is the addend of encoder k's max-pool backward."""
        sv = self.saved
        flat = self.alloc_grads(g_logits.device)
        self._begin_pass(g_logits.shape[0], g_logits.device, backward=True)
        g = self.head_backward(sv["head"], g_logits)
        gS: List[Optional[Tensor]] = [None] * 4
        for k in (1, 2, 3, 4):
            gS[k - 1] = g
            L1, L2 = sv[f"decoder{k}"]
            self._tag(f"decoder{k}")
            gd = torch.empty(L2.y.shape, dtype=self.T, device=g.device)
            self.be.upsample_bwd(g, gd)
            g1 = self.bwd_layer(L2, gd, True, prev=L1)
            g = self.bwd_layer(L1, g1, True)
        L1, L2 = sv["bottleneck"]
        g = self.bwd_layer(L1, self.bwd_layer(L2, g, True, prev=L1), True)
        self._flush_bucket("bottleneck.bottleneckconv1.weight")
        self._early_unpack()
        for i in (3, 2, 1, 0):
            e, pooled = sv[f"pool{i + 1}"]
            ge = torch.empty(e.shape, dtype=self.T, device=e.device)
            self.be.pool_bwd(e, g, gS[i], ge, 3)                         # + the skip's gradient
            L1, L2 = sv[f"encoder{i + 1}"]
            g1 = self.bwd_layer(L2, ge, True, prev=L1)
            g = self.bwd_layer(L1, g1, i > 0)
        self._finish_backward()
        return flat
