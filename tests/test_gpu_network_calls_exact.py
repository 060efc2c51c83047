"""Every convolution, weight gradient and max-pool call a training step of the networks makes, replayed bit for bit
against fp64 at the buffer layouts the engine hands the kernels.

The hand-picked cases of test_gpu_conv_exact.py and test_gpu_gn_exact.py use a synthetic layout (channel pitch C + 16,
a channel offset of at most 16).  The networks hand the kernels other views: the right half of a [up | skip] concat
buffer (pitch 2C at channel offset C), concat halves as the addend of a data gradient, the permuted NCDHW image, and
weights packed for each layer's own voxel count.  This file records what the engine actually launches and replays it.

1. Record.  `Recorder` wraps the backend (installed with runtime._set_backend_for_testing) and records every conv,
   conv_bwdstats, wgrad, pool_fwd and pool_bwd call of one eager training step (train mode, dropout on): per tensor
   its sizes, strides, storage offset, storage length, dtype and data_ptr % 512; per packed weight its kind, which,
   dims, layout code and shapes; whether bias, statistics and addend are present; the GroupNorm descriptor of
   conv_bwdstats; the kernel family (conv_path / wgrad_path on the live arguments).  Engine._tag labels each call
   with its network block.  Calls are deduplicated on everything recorded except the labels.
2. Replay.  Each unique call runs again on operands from the exact grids of test_gpu_conv_exact.py, every tensor
   rebuilt with as_strided at its recorded layout inside one allocation with a guard band of whole 512-byte blocks
   on each side (so the view keeps its recorded alignment).  Inputs hold IN_FILL everywhere outside the view, outputs
   the NaN pattern.  Outputs must equal the fp64 reference rounded to their dtype bit for bit, nothing outside an
   output view may change and no input may change.  Forward statistics are compared bit for bit where the operands
   prove every fp32 partial exact (stats_exact), else within the fp32 chain bound of stats_chain.

The CPU part records the same steps on the emulated backend (tests/emu_backend.py) at small sizes and checks the
recorder, the rebuilt layouts and the checkers; the GPU part is marked `gpu`."""
import math
import time
from collections import namedtuple

import pytest
import torch

from emu_backend import DOWN, UP
from test_gpu_conv_exact import (CONV_PATHS, GUARD, IN_FILL, OUT_BITS, bwdstats_want, check_stats,
                                 conv_quantum, exact_bound, first_mismatch, grid, ref_conv, ref_wgrad, stats_chain)
from test_gpu_gn_exact import pool_input, pool_ref

OPS = ("conv", "conv_bwdstats", "wgrad", "pool_fwd", "pool_bwd")
FAMILY = {"conv": "conv", "conv_bwdstats": "bwdstats", "wgrad": "wgrad", "pool_fwd": "pool", "pool_bwd": "pool"}
BLOCK = 512                   # bytes: the alignment a rebuilt view keeps
GUARD_BLOCKS = 2              # guard band before and after every rebuilt storage, in blocks
DTYPES = {"bfloat16": torch.bfloat16, "float32": torch.float32, "float64": torch.float64}
FILL_BITS = {**OUT_BITS, torch.float64: (torch.int64, 0x7FF80000DEADBEEF)}     # NaN payloads of a fresh output

# forward statistics that are not compared with fp64, by kernel family, with the reason.  Every family the networks
# reach has a chain bound in stats_chain, so none is exempt; a family added to the library must be derived there or
# listed here.
STATS_UNCHECKED = {}

# the steps: net, constructor arguments, batch, spatial size
WORKLOADS = {
    "vnet3d_96": ("VNet3d", (1, 2), 2, (96, 96, 96)),
    "vnet3d_128x112": ("VNet3d", (1, 2), 1, (128, 112, 112)),
    "unet3d_128": ("UNet3d", (1, 4), 1, (128, 128, 128)),
    "unet3d_128x112": ("UNet3d", (1, 4), 1, (128, 112, 112)),
    "unet2d_512": ("UNet2d", (1, 1), 8, (512, 512)),
    "vnet2d_512": ("VNet2d", (1, 2), 8, (512, 512)),
    "vnet2d_128x96": ("VNet2d", (1, 2), 2, (128, 96)),
    "resnet3d_96": ("ResNet3d", (1, 4), 2, (96, 96, 96)),
    "resnet2d_64": ("ResNet2d", (1, 10), 128, (64, 64)),
}
CPU_WORKLOADS = {
    "vnet3d_32": ("VNet3d", (1, 2), 2, (32, 32, 32)),
    "unet2d_64": ("UNet2d", (1, 1), 2, (64, 64)),
    "resnet3d_32": ("ResNet3d", (1, 4), 2, (32, 32, 32)),
}
FIRST_LAYERS = {"in_tr.conv1.weight", "in_tr.conv2.weight", "encoder1.enc1conv1.weight"}   # they read the image
HEADS = {"out_tr.conv.weight", "conv.weight"}                                           # the fused segmentation heads

TRec = namedtuple("TRec", "sizes strides offset storage dtype align")
WRec = namedtuple("WRec", "kind which dims code tshape tdtype src")
Call = namedtuple("Call", "op kind dims path t w bias stats gn")     # t: ((role, TRec | None), ...)


# ---------------------------------------------------------------------------------------------------------- record
def trec(t):
    if t is None:
        return None
    return TRec(tuple(t.shape), tuple(t.stride()), t.storage_offset(), t.untyped_storage().nbytes() // t.element_size(),
                str(t.dtype).split(".")[-1], t.data_ptr() % BLOCK)


def pitch(r):
    """channel pitch ld and channel offset of an (N, D, H, W, C) view"""
    ld = r.strides[3]
    return ld, r.offset % ld


class Recorder:
    """The backend, recording the conv / conv_bwdstats / wgrad / pool calls and forwarding them unchanged.  `tag` is
    set by Engine._tag to the block the next launches belong to.  On the emulated backend, whose packed operands are
    plain tensors, the pack calls are wrapped too so that each operand's kind, which and dims are known."""

    def __init__(self, inner, names=None, ops=OPS, hook=None):
        self.inner = inner
        self.tag = "other"
        self.calls = []
        self.names = names or {}              # data_ptr of a parameter -> its name (labels only)
        self.ops = ops                        # the entry points recorded
        self.hook = hook                      # (recorder, op, args, kwargs) -> record dict; default: _record
        self._packed = {}                     # emulated backend: id(packed tensor) -> (packed, src, kind, which, dims)

    def __getattr__(self, name):
        fn = getattr(self.inner, name)
        if name in self.ops:
            def record(*a, **k):
                self.calls.append(self._record(name, a) if self.hook is None else self.hook(self, name, a, k))
                return fn(*a, **k)
            return record
        if name in ("pack_weight", "pack_many", "pack_plan") and not hasattr(self.inner, "conv_path"):
            def pack(*a, **k):
                out = fn(*a, **k)
                reqs = [a[:5]] if name == "pack_weight" else a[0]
                outs = [out] if name == "pack_weight" else (out if name == "pack_many" else out.outs)
                for (w, kind, which, _, dims, *_), o in zip(reqs, outs):
                    self._packed[id(o)] = (o, w, kind, which, dims)
                return out
            return pack
        return fn

    def _wrec(self, wpk):
        if hasattr(wpk, "code"):
            return WRec(wpk.kind, wpk.which, wpk.dims, wpk.code, tuple(wpk.t.shape), str(wpk.t.dtype).split(".")[-1],
                        tuple(wpk.src.shape)), wpk.src
        o, src, kind, which, dims = self._packed[id(wpk)]
        return WRec(kind, which, dims, None, tuple(o.shape), str(o.dtype).split(".")[-1], tuple(src.shape)), src

    def _record(self, op, a):
        inner, w, src, bias, stats, gn, path = self.inner, None, None, False, False, None, None
        if op == "conv":
            kind, dims, x, wpk, b, y, st, addend = a
            t = (("x", x), ("y", y), ("addend", addend))
            w, src = self._wrec(wpk)
            bias, stats = b is not None, st is not None
            if hasattr(inner, "conv_path"):
                path = inner.conv_path(kind, dims, x, wpk, y, addend)
        elif op == "conv_bwdstats":
            kind, dims, x, wpk, y, addend, yfwd, g, sums = a
            t = (("x", x), ("y", y), ("addend", addend), ("yfwd", yfwd))
            w, src = self._wrec(wpk)
            gn = (g[4], g[5], g[6], g[3] is not None)
            if hasattr(inner, "conv_path"):
                path = inner.conv_path(kind, dims, x, wpk, y, addend)
        elif op == "wgrad":
            kind, dims, A, B, dwp = a
            t = (("a", A), ("b", B))
            w = tuple(dwp.shape)
            if hasattr(inner, "wgrad_path"):
                path = inner.wgrad_path(kind, dims, A, B)
        elif op == "pool_fwd":
            x, out, dims = a
            kind, t = None, (("x", x), ("out", out))
        else:
            x, g_out, addend, g_x, dims = a
            kind, t = None, (("x", x), ("g_out", g_out), ("addend", addend), ("g_x", g_x))
        sig = Call(op, kind, dims, path, tuple((r, trec(v)) for r, v in t), w, bias, stats, gn)
        return {"sig": sig, "tag": self.tag, "weight": None if src is None else self.names.get(src.data_ptr())}


def record_step(backend, workload, precision, device, table=WORKLOADS, ops=OPS, hook=None):
    """one eager training step of the workload in train mode (dropout on) -> (recorded calls, parameter names, model);
    `ops` and `hook` go to Recorder"""
    import pytorchdeeplearing_b200 as b200
    from pytorchdeeplearing_b200 import runtime
    net, args, n, sp = table[workload]
    ncls = args[1]
    prev = runtime.get_precision()
    b200.set_precision(precision)
    torch.manual_seed(0)
    m = getattr(b200, net)(*args)
    m.apply(b200.initialize_weights)
    m = m.to(device).train()
    g = torch.Generator().manual_seed(1)
    x = torch.randn((n, args[0]) + sp, generator=g)
    if net.startswith("ResNet"):
        y, loss = torch.randint(0, ncls, (n,), generator=g), b200.MutilCrossEntropyLoss(torch.ones(ncls, device=device))
    elif ncls == 1:
        y, loss = (torch.rand((n,) + sp, generator=g) > 0.7).long(), b200.BinaryDiceLoss()
    else:
        y, loss = torch.randint(0, ncls, (n,) + sp, generator=g), b200.MutilDiceLoss(torch.ones(ncls, device=device))
    rec = Recorder(backend, {p.data_ptr(): name for name, p in m.named_parameters()}, ops, hook)
    runtime._set_backend_for_testing(rec)
    try:
        out = m(x.to(device))
        logits = out[0] if isinstance(out, tuple) else out
        loss(logits, y.to(device)).backward()
        if device == "cuda":
            torch.cuda.synchronize()
        assert all(p.grad is not None for p in m.parameters())
    finally:
        runtime._set_backend_for_testing(None)
        b200.set_precision(prev)
    return rec.calls, [name for name, _ in m.named_parameters()], m


def unique_calls(calls):
    """signature -> the tags of all its occurrences (in order of first appearance)"""
    u = {}
    for c in calls:
        tags = u.setdefault(c["sig"], [])
        if c["tag"] not in tags:
            tags.append(c["tag"])
    return u


# ---------------------------------------------------------------------------------------------------------- rebuild
class Rebuilt:
    """a recorded view rebuilt with as_strided inside one allocation: the recorded storage with GUARD_BLOCKS blocks of
    512 bytes before and after it, placed at the recorded storage's own remainder mod 512 past a block boundary (zero
    for CUDA allocations), so that the view's address has its recorded remainder mod 512.  Every element outside the
    view holds `fill` (a float), or the NaN pattern of the dtype (fill=None)."""

    def __init__(self, r, fill=None, device="cuda"):
        self.r, self.dtype = r, DTYPES[r.dtype]
        es = torch.empty((), dtype=self.dtype).element_size()
        gb = GUARD_BLOCKS * BLOCK
        assert gb % BLOCK == 0
        mis = (r.align - r.offset * es) % BLOCK         # byte remainder of the recorded storage's address
        assert mis % es == 0
        self.buf = torch.empty(BLOCK // es + (gb + mis) // es + r.storage + gb // es, dtype=self.dtype, device=device)
        a0 = (-self.buf.data_ptr() % BLOCK) // es         # first 512-aligned element
        self.s0 = a0 + (gb + mis) // es                    # first element of the rebuilt storage
        self.guard = (a0 * es, gb + mis, gb)
        if fill is None:
            ib, pat = FILL_BITS[self.dtype]
            self.buf.view(ib).fill_(pat)
        else:
            self.buf.fill_(fill)
        self.view = self.buf.as_strided(r.sizes, r.strides, self.s0 + r.offset)
        assert (self.buf.data_ptr() + a0 * es) % BLOCK == 0
        assert self.view.data_ptr() % BLOCK == r.align, "rebuilt view lost its alignment"
        self.before = None

    def set(self, v):
        self.view.copy_(v.to(self.dtype))
        return self

    def snapshot(self):
        self.before = self.buf.clone()
        return self

    def changed(self, inside=False):
        """None, or a description of the first element whose bits changed since the snapshot (outside the view only,
        unless `inside`)"""
        ib = FILL_BITS[self.dtype][0]
        ne = self.buf.view(ib) != self.before.view(ib)
        if not inside:
            ne.as_strided(self.r.sizes, self.r.strides, self.s0 + self.r.offset).fill_(False)
        if not bool(ne.any()):
            return None
        i = int(ne.nonzero()[0]) - self.s0
        if i < 0 or i >= self.r.storage:
            return f"element {i} of the storage, in the guard band"
        if len(self.r.strides) != 5:
            return f"element {i} of the storage, outside the view"
        ld, off = pitch(self.r)
        return (f"element {i} of the storage (row {i // ld}, channel {i % ld - off} of the view's pitch), in the "
                f"{'storage' if inside else 'storage outside the view (other concat half or pitch gap)'}")


# ---------------------------------------------------------------------------------------------------------- checks
def check_out(rb, want, what):
    """None, or a message: the view bitwise against want (N,D,H,W,C), then everything outside the view unchanged"""
    msg = first_mismatch(rb.view, want.to(rb.dtype))
    if msg is not None:
        return f"{what}: inside the view: {msg}"
    pos = rb.changed()
    return None if pos is None else f"{what}: written outside the view: {pos}"


def check_in(rb, what):
    pos = rb.changed(inside=True)
    return None if pos is None else f"{what}: input changed: {pos}"


def stats_exact(path, v, q):
    """do the operands prove every partial of the statistics of v exact (v a multiple of q)?  GENERIC adds at most 4
    values of a column in fp32 and the rest in fp64 (conv_generic.cu:186-216); every other family forms fp32 partial
    sums of subsets of one (n, c)'s values, so the whole sum must stay below 2^24 quanta."""
    a = v.abs()
    dims = tuple(range(1, v.dim() - 1))
    q2 = q * q
    if path == "GENERIC":
        m = float(a.max())
        return 4 * m < 2 ** 24 * q and 4 * m * m < 2 ** 24 * q2 and float((v * v).sum(dims).max()) < 2 ** 53 * q2
    return float(a.sum(dims).max()) < 2 ** 24 * q and float((v * v).sum(dims).max()) < 2 ** 24 * q2


class Log:
    """per (workload, precision, family): failures, and the statistics cases by how they were checked"""

    def __init__(self, label):
        self.label, self.failures, self.paths = label, [], set()
        self.stats = {"bitwise": 0, "bound": 0, "unchecked": 0}
        self.generic_bitwise = 0

    def fail(self, sig, tags, msg):
        self.failures.append(f"{self.label} {sig.op} path={sig.path} tags={','.join(tags)}: {msg}")


# ---------------------------------------------------------------------------------------------------------- CPU part
_CPU_RECORDINGS = {}


def _cpu_recording(workload):
    if workload not in _CPU_RECORDINGS:
        torch.set_num_threads(max(1, min(8, torch.get_num_threads())))
        from test_resnet_cpu import ClsEmuBackend           # the emulated backend plus the classifier head
        _CPU_RECORDINGS[workload] = record_step(ClsEmuBackend(), workload, "fp32", "cpu", CPU_WORKLOADS)
    return _CPU_RECORDINGS[workload]


@pytest.mark.parametrize("workload", sorted(CPU_WORKLOADS))
def test_call_counts_follow_the_layer_program(workload):
    """one forward conv per conv weight, one data gradient per weight that does not read the image, one wgrad per
    weight (per block); the heads run through their own kernels on the emulated backend too"""
    calls, names, m = _cpu_recording(workload)
    params = dict(m.named_parameters())
    convw = [nm for nm in names if params[nm].dim() >= 3 and nm not in HEADS]
    fwd, dgrad = {}, {}
    for c in calls:
        s = c["sig"]
        if s.op in ("conv", "conv_bwdstats"):
            assert c["weight"] is not None
            d = fwd if s.w.which == "fwd" else dgrad
            d[c["weight"]] = d.get(c["weight"], 0) + 1
    assert fwd == {nm: 1 for nm in convw}
    assert dgrad == {nm: 1 for nm in convw if nm not in FIRST_LAYERS}
    per_block = {}
    for nm in convw:
        per_block[nm.split(".")[0]] = per_block.get(nm.split(".")[0], 0) + 1
    wg = {}
    for c in calls:
        if c["sig"].op == "wgrad":
            wg[c["tag"]] = wg.get(c["tag"], 0) + 1
    assert wg == per_block
    n_pool = sum(c["sig"].op.startswith("pool") for c in calls)
    assert n_pool == (8 if workload.startswith("unet") else 0)


def test_skip_halves_arrive_as_concat_views():
    """VNet3d: every down convolution reads the right half of a [up | skip] concat (pitch 2C, offset C), and every
    down convolution's data gradient adds the skip half of a concat gradient; UNet2d: pool_fwd reads the encoder
    output at offset C of its concat and pool_bwd adds the other concat gradient's skip half"""
    calls, _, _ = _cpu_recording("vnet3d_32")
    downs = [c for c in calls if c["sig"].op == "conv" and c["sig"].kind == DOWN and c["sig"].w.which == "fwd"]
    assert len(downs) == 4
    for c in downs:
        x = dict(c["sig"].t)["x"]
        assert pitch(x) == (2 * x.sizes[-1], x.sizes[-1]), c
    dd = [c for c in calls if c["sig"].op == "conv" and c["sig"].w.kind == DOWN and c["sig"].w.which == "dgrad"]
    assert len(dd) == 4
    for c in dd:
        a = dict(c["sig"].t)["addend"]
        assert a is not None and pitch(a) == (2 * a.sizes[-1], a.sizes[-1]), c
    calls, _, _ = _cpu_recording("unet2d_64")
    for c in calls:
        if c["sig"].op.startswith("pool"):
            t = dict(c["sig"].t)
            assert pitch(t["x"]) == (2 * t["x"].sizes[-1], t["x"].sizes[-1]), c
            if c["sig"].op == "pool_bwd":
                assert pitch(t["addend"]) == (2 * t["addend"].sizes[-1], t["addend"].sizes[-1]), c


@pytest.mark.parametrize("workload", sorted(CPU_WORKLOADS))
def test_rebuilt_views_keep_the_recorded_layout(workload):
    calls, _, _ = _cpu_recording(workload)
    seen = set()
    for sig in unique_calls(calls):
        for _, r in sig.t:
            if r is None or r in seen:
                continue
            seen.add(r)
            rb = Rebuilt(r, fill=IN_FILL, device="cpu")
            assert tuple(rb.view.shape) == r.sizes and tuple(rb.view.stride()) == r.strides
            assert rb.view.storage_offset() == rb.s0 + r.offset
            assert rb.view.data_ptr() % BLOCK == r.align
            assert rb.s0 * rb.buf.element_size() - rb.guard[0] == rb.guard[1] and rb.guard[2] % BLOCK == 0
            assert rb.buf.numel() - rb.s0 - r.storage >= rb.guard[2] // rb.buf.element_size()


def _skip_half_rec():
    calls, _, _ = _cpu_recording("vnet3d_32")
    c = next(c for c in calls if c["sig"].op == "conv" and c["sig"].kind == DOWN and c["sig"].w.which == "fwd")
    x = dict(c["sig"].t)["x"]
    return x._replace(dtype="bfloat16", storage=x.storage, align=0)


def _want(r):
    g = torch.Generator().manual_seed(9)
    return grid(r.sizes, 200, 4, g).float().bfloat16()


def test_checker_reports_one_ulp():
    r = _skip_half_rec()
    rb = Rebuilt(r, device="cpu").snapshot()
    want = _want(r)
    rb.view.copy_(want)
    assert check_out(rb, want, "exact") is None
    rb.view.view(torch.int16)[1, 2, 3, 4, 7] += 1
    assert "(1, 2, 3, 4, 7)" in check_out(rb, want, "one ulp")


def test_checker_reports_a_byte_in_the_other_concat_half():
    r = _skip_half_rec()
    rb = Rebuilt(r, device="cpu").snapshot()
    want = _want(r)
    rb.view.copy_(want)
    ld, off = pitch(r)
    assert off == r.sizes[-1] and ld == 2 * off
    rb.buf.view(torch.uint8)[2 * (rb.s0 + 5 * ld + 3)] ^= 1      # one byte of channel 3 of row 5: the left half
    msg = check_out(rb, want, "other half")
    assert msg is not None and "outside the view" in msg and "other concat half" in msg


def test_checker_reports_a_view_shifted_by_8_channels():
    r = _skip_half_rec()
    rb = Rebuilt(r, device="cpu").snapshot()
    want = _want(r)
    rb.buf.as_strided(r.sizes, r.strides, rb.s0 + r.offset - 8).copy_(want)
    msg = check_out(rb, want, "shifted")
    assert msg is not None and "inside the view" in msg
    rb.view.copy_(want)                                           # the right values, plus the stray 8-channel stores
    msg = check_out(rb, want, "shifted")
    assert msg is not None and "outside the view" in msg


def test_checker_reports_rounding_from_an_unrounded_fp32_sum():
    """1 + 2^-8 + 2^-30 rounds up to bf16 1 + 2^-7; its fp32 sum 1 + 2^-8 is a tie that rounds down to 1"""
    r = _skip_half_rec()
    rb = Rebuilt(r, device="cpu").snapshot()
    want = torch.ones(r.sizes, dtype=torch.bfloat16)          # the exact sums, rounded once to nearest even
    want[0, 1, 2, 3, 4] = 1 + 2.0 ** -7
    terms = (torch.ones(r.sizes, dtype=torch.float32), torch.full(r.sizes, 2.0 ** -8), torch.zeros(r.sizes))
    terms[2][0, 1, 2, 3, 4] = 2.0 ** -30
    fp32_sum = terms[0] + terms[1] + terms[2]
    rb.view.copy_(fp32_sum.bfloat16())
    assert "(0, 1, 2, 3, 4)" in check_out(rb, want, "fp32 sum")


def test_stats_chain_covers_every_conv_family():
    for p in CONV_PATHS:
        assert p in STATS_UNCHECKED or stats_chain(p, 2, (6, 8, 16), 64) >= 4


# ---------------------------------------------------------------------------------------------------------- GPU part
@pytest.fixture(scope="module")
def be():
    from pytorchdeeplearing_b200._abi import CudaBackend
    return CudaBackend()


_RECORDINGS = {}


def _recording(be, workload, precision):
    key = (workload, precision)
    if key not in _RECORDINGS:
        calls, _, m = record_step(be, workload, precision, "cuda")
        del m
        _RECORDINGS[key] = calls
    return _RECORDINGS[key]


def _dt(s):
    return DTYPES[s]


def _ys(r):
    return r.sizes[1:4]


def replay_conv(be, sig, gen, log, sms):
    T = dict(sig.t)
    xr, yr, ar = T["x"], T["y"], T["addend"]
    w = sig.w
    x_full = sig.path == "STEM_MMA" and xr.dtype == "float32" and yr.dtype == "bfloat16"
    cs = dict(kind=w.kind, which=w.which, dims=sig.dims, x_full=x_full)
    co = yr.sizes[-1]
    x = grid(xr.sizes, 4, 2, gen)
    if x_full:
        mag = torch.rand(xr.sizes, generator=gen, device="cuda", dtype=torch.float64) * (4 - 0.125) + 0.125
        sign = torch.randint(0, 2, mag.shape, generator=gen, device="cuda").double() * 2 - 1
        x = (mag * sign).float().double()
    wt = grid(w.src, 8, 5, gen)
    bias = grid((co,), 16, 7, gen) if sig.bias else None
    addend = grid(ar.sizes, 128, 7, gen) if ar is not None else None
    assert exact_bound(cs, x, wt, bias, addend) < 2 ** 20 * conv_quantum(cs), "exactness precondition"
    xk = x.float().bfloat16().double() if x_full else x
    v, yref = ref_conv(cs, xk, wt, bias, addend)
    gx = Rebuilt(xr, IN_FILL).set(x).snapshot()
    ga = None if ar is None else Rebuilt(ar, IN_FILL).set(addend).snapshot()
    gy = Rebuilt(yr).snapshot()
    wp = be.pack_weight(wt.float(), w.kind, w.which, _dt(w.tdtype), w.dims, vox=math.prod(_ys(yr)))
    assert (wp.code, tuple(wp.t.shape)) == (w.code, w.tshape), "re-packed weight differs from the recorded one"
    assert be.conv_path(sig.kind, sig.dims, gx.view, wp, gy.view, None if ga is None else ga.view) == sig.path
    gs = None
    n = yr.sizes[0]
    if sig.stats:
        gs = torch.full((2 * GUARD + n * co * 2,), float("nan"), dtype=torch.float64, device="cuda")
        gs[GUARD:-GUARD] = 0
    be.conv(sig.kind, sig.dims, gx.view, wp, None if bias is None else bias.float(), gy.view,
            None if gs is None else gs[GUARD:-GUARD].view(n, co, 2), None if ga is None else ga.view)
    torch.cuda.synchronize()
    msgs = [check_out(gy, yref.float(), "y"), check_in(gx, "x")]
    if ga is not None:
        msgs.append(check_in(ga, "addend"))
    if gs is not None:
        if not bool(torch.cat([gs[:GUARD], gs[-GUARD:]]).isnan().all()):
            msgs.append("statistics guard band written")
        got = gs[GUARD:-GUARD].view(n, co, 2)
        if sig.path in STATS_UNCHECKED:
            log.stats["unchecked"] += 1
        elif stats_exact(sig.path, v, conv_quantum(cs)):
            log.stats["bitwise"] += 1
            log.generic_bitwise += sig.path == "GENERIC"
            want = torch.stack([v.sum((1, 2, 3)), (v * v).sum((1, 2, 3))], -1)
            if not torch.equal(got, want):
                nn_, c, k = (got != want).nonzero()[0].tolist()
                msgs.append(f"statistics (bitwise) of (n, c) = ({nn_}, {c})[{k}]: {float(got[nn_, c, k])!r}, "
                            f"fp64 {float(want[nn_, c, k])!r}")
        else:
            log.stats["bound"] += 1
            chain = stats_chain(sig.path, n, _ys(yr), co, up=sig.kind == UP, kind=sig.kind, dims=sig.dims, sms=sms)
            try:
                check_stats(got, v, chain, "statistics")
            except AssertionError as e:
                msgs.append(str(e))
    return [m for m in msgs if m is not None]


def replay_bwdstats(be, sig, gen, log, sms):
    T = dict(sig.t)
    xr, yr, ar, fr = T["x"], T["y"], T["addend"], T["yfwd"]
    w = sig.w
    cs = dict(kind=w.kind, which=w.which, dims=sig.dims, x_full=False)
    n, co = yr.sizes[0], yr.sizes[-1]
    vox, groups, eps, _ = sig.gn
    assert vox == math.prod(_ys(yr)) and fr.sizes == yr.sizes
    x = grid(xr.sizes, 4, 2, gen)
    wt = grid(w.src, 8, 5, gen)
    addend = grid(ar.sizes, 128, 7, gen) if ar is not None else None
    assert exact_bound(cs, x, wt, None, addend) < 2 ** 20 * conv_quantum(cs), "exactness precondition"
    g_bf = ref_conv(cs, x, wt, None, addend)[1].float().bfloat16()
    yfwd = torch.randn(fr.sizes, generator=gen, device="cuda").bfloat16()
    yf = yfwd.double()
    stats = torch.stack([yf.sum((1, 2, 3)), (yf * yf).sum((1, 2, 3))], -1).contiguous()
    gamma = (1 + 0.2 * torch.randn(co, generator=gen, device="cuda")).float()
    beta = (0.3 * torch.randn(co, generator=gen, device="cuda")).float()
    scale = ((torch.rand((n, co), generator=gen, device="cuda") > 0.2).float() / 0.8).float()
    gx = Rebuilt(xr, IN_FILL).set(x).snapshot()
    ga = None if ar is None else Rebuilt(ar, IN_FILL).set(addend).snapshot()
    gf = Rebuilt(fr, IN_FILL).set(yfwd).snapshot()
    wp = be.pack_weight(wt.float(), w.kind, w.which, _dt(w.tdtype), w.dims, vox=math.prod(_ys(yr)))
    assert (wp.code, tuple(wp.t.shape)) == (w.code, w.tshape), "re-packed weight differs from the recorded one"
    av = None if ga is None else ga.view
    assert be.conv_path(sig.kind, sig.dims, gx.view, wp, Rebuilt(yr).view, av) == sig.path
    chain = stats_chain(sig.path, n, _ys(yr), co, sms=sms)
    msgs = []
    for sc in (None, scale):
        gy = Rebuilt(yr).snapshot()
        assert be.conv_bwdstats_ok(sig.kind, sig.dims, gx.view, wp, gy.view, av, gf.view)
        sbuf = torch.full((2 * GUARD + n * co * 3,), float("nan"), dtype=torch.float64, device="cuda")
        sbuf[GUARD:-GUARD] = 0
        sums = sbuf[GUARD:-GUARD].view(n, co, 3)
        be.conv_bwdstats(sig.kind, sig.dims, gx.view, wp, gy.view, av, gf.view,
                         (stats, gamma, beta, sc, vox, groups, eps), sums)
        torch.cuda.synchronize()
        what = "no scale" if sc is None else "dropout scale"
        msgs += [check_out(gy, g_bf, f"g ({what})"), check_in(gx, "dy"), check_in(gf, "yfwd")]
        if ga is not None:
            msgs.append(check_in(ga, "addend"))
        if not bool(torch.cat([sbuf[:GUARD], sbuf[-GUARD:]]).isnan().all()):
            msgs.append(f"sums guard band written ({what})")
        if float(sums[..., 2].abs().max()) != 0.0:
            msgs.append(f"sums[..., 2] written ({what})")
        s0, t0, s1, t1 = bwdstats_want(g_bf, yf, stats, gamma, beta, sc, groups, eps, chain)
        for k, (want, tol) in enumerate(((s0, t0), (s1, t1))):
            bad = (sums[..., k] - want).abs() > tol
            if bool(bad.any()):
                nn_, c = bad.nonzero()[0].tolist()
                msgs.append(f"sums[{nn_}][{c}][{k}] ({what}) = {float(sums[nn_, c, k])!r}, fp64 "
                            f"{float(want[nn_, c])!r}, bound {float(tol[nn_, c]):.3g}")
        log.stats["bound"] += 1
    return [m for m in msgs if m is not None]


def replay_wgrad(be, sig, gen, log, sms):
    T = dict(sig.t)
    ar, br = T["a"], T["b"]
    a = torch.randint(-1, 2, ar.sizes, generator=gen, device="cuda").double()
    b = torch.randint(-1, 2, br.sizes, generator=gen, device="cuda").double() * 0.5
    ws = dict(kind=sig.kind, dims=sig.dims, ca=ar.sizes[-1], cb=br.sizes[-1])
    assert 2 * float(ref_wgrad(ws, a.abs(), b.abs()).max()) < 2 ** 23, "exactness precondition"
    want = ref_wgrad(ws, a, b).float()
    assert tuple(want.shape) == sig.w, (tuple(want.shape), sig.w)
    ga = Rebuilt(ar, IN_FILL).set(a).snapshot()
    gb = Rebuilt(br, IN_FILL).set(b).snapshot()
    buf = torch.full((2 * GUARD + want.numel(),), float("nan"), device="cuda")
    buf[GUARD:-GUARD] = 0
    dwp = buf[GUARD:-GUARD].view(want.shape)
    assert be.wgrad_path(sig.kind, sig.dims, ga.view, gb.view) == sig.path
    msgs = []
    for k in (1, 2):                                         # the second call accumulates
        be.wgrad(sig.kind, sig.dims, ga.view, gb.view, dwp)
        torch.cuda.synchronize()
        m = first_mismatch(dwp.view(want.shape + (1, 1)), (k * want).view(want.shape + (1, 1)))
        if m is not None:
            msgs.append(f"dwp (call {k}; index (t, ca, cb, -, -)): {m}")
    if not bool(torch.cat([buf[:GUARD], buf[-GUARD:]]).isnan().all()):
        msgs.append("dwp guard band written")
    msgs += [check_in(ga, "a"), check_in(gb, "b")]
    return [m for m in msgs if m is not None]


def replay_pool(be, sig, gen, log, sms):
    T = dict(sig.t)
    xr = T["x"]
    n, sp, c = xr.sizes[0], xr.sizes[1:4], xr.sizes[-1]
    x, _ = pool_input(sig.dims, n, sp, c, gen)
    gx = Rebuilt(xr, IN_FILL).set(x).snapshot()
    msgs = []
    if sig.op == "pool_fwd":
        out = Rebuilt(T["out"]).snapshot()
        go = torch.zeros(T["out"].sizes, dtype=torch.float64, device="cuda")
        be.pool_fwd(gx.view, out.view, sig.dims)
        torch.cuda.synchronize()
        msgs.append(check_out(out, pool_ref(sig.dims, x, go)[0].float(), "pooled"))
    else:
        gor, adr, gxr = T["g_out"], T["addend"], T["g_x"]
        go = torch.randint(-8, 9, gor.sizes, generator=gen, device="cuda").double() / 8
        ggo = Rebuilt(gor, IN_FILL).set(go).snapshot()
        add = None
        gad = None
        if adr is not None:
            add = torch.randint(-8, 9, adr.sizes, generator=gen, device="cuda").double() / 16
            gad = Rebuilt(adr, IN_FILL).set(add).snapshot()
        gxo = Rebuilt(gxr).snapshot()
        be.pool_bwd(gx.view, ggo.view, None if gad is None else gad.view, gxo.view, sig.dims)
        torch.cuda.synchronize()
        want = pool_ref(sig.dims, x, go)[1] + (add if add is not None else 0)
        msgs += [check_out(gxo, want.float(), "g_x"), check_in(ggo, "g_out")]
        if gad is not None:
            msgs.append(check_in(gad, "addend"))
    msgs.append(check_in(gx, "x"))
    return [m for m in msgs if m is not None]


REPLAY = {"conv": replay_conv, "bwdstats": replay_bwdstats, "wgrad": replay_wgrad, "pool": replay_pool}


def required_facts(family, workload, precision, calls):
    """what the replays of a family must include: -> [(description, holds)]"""
    facts = []
    if (workload, precision, family) == ("vnet3d_96", "bf16", "conv"):
        def xs(c):
            return dict(c.t)
        concat_off64 = any(r is not None and role in ("x", "y") and pitch(r)[0] == 2 * r.sizes[-1]
                           and pitch(r)[1] == r.sizes[-1] >= 64 for c in calls for role, r in c.t)
        addend_half = any(c.w.which == "dgrad" and xs(c)["addend"] is not None
                          and pitch(xs(c)["addend"])[0] == 2 * xs(c)["addend"].sizes[-1] for c in calls)
        ws_small = any(c.path == "HALO_WS" and _ys(xs(c)["y"]) in ((6, 6, 6), (12, 12, 12)) for c in calls)
        facts += [("a view with ld = 2C at channel offset C >= 64", concat_off64),
                  ("a data gradient whose addend is a concat half", addend_half),
                  ("a HALO_WS call at 6^3 or 12^3", ws_small)]
    return facts


GPU_CASES = [(w, p, f) for w in WORKLOADS for p in ("bf16", "fp32") for f in ("conv", "bwdstats", "wgrad", "pool")
             if (f != "pool" or w.startswith("unet")) and (f != "bwdstats" or p == "bf16")]


@pytest.mark.gpu
@pytest.mark.parametrize("workload,precision,family", GPU_CASES, ids=["-".join(c) for c in GPU_CASES])
def test_network_calls_exact(be, workload, precision, family):
    t0 = time.time()
    calls = _recording(be, workload, precision)
    uniq = {s: tags for s, tags in unique_calls(calls).items() if FAMILY[s.op] == family}
    n_rec = sum(FAMILY[c["sig"].op] == family for c in calls)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    log = Log(f"{workload} {precision}")
    gen = torch.Generator(device="cuda")
    for i, (sig, tags) in enumerate(uniq.items()):
        gen.manual_seed(1000 + i)
        log.paths.add(sig.path)
        try:
            for m in REPLAY[family](be, sig, gen, log, sms):
                log.fail(sig, tags, m)
        except AssertionError as e:
            log.fail(sig, tags, f"{e}")
        torch.cuda.empty_cache()
    for what, holds in required_facts(family, workload, precision, list(uniq)):
        if not holds:
            log.failures.append(f"{log.label} {family}: no replayed call has {what}")
    if (workload, precision, family) == ("vnet3d_96", "fp32", "conv") and log.generic_bitwise == 0:
        log.failures.append(f"{log.label}: no GENERIC forward statistics were checked bit for bit")
    st = log.stats
    print(f"\n{workload:15s} {precision:5s} {family:9s} recorded {n_rec:4d} unique {len(uniq):3d} "
          f"families {','.join(sorted(p for p in log.paths if p)) or '-'} "
          f"stats bitwise {st['bitwise']} bound {st['bound']} unchecked {st['unchecked']} "
          f"({time.time() - t0:.1f} s)")
    assert not log.failures, "\n".join(log.failures)
