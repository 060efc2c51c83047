"""Per-kernel timings at the VNet3d 96^3 / batch-2 layer shapes, through the C ABI (one GPU).

    python tools/microbench_ops.py [--reps 20] [--only stem,stemgn,gn,pack,wgrad,conv]

Every op is timed with CUDA events on the current stream, once with a warm L2 (back-to-back launches) and
once "cold" (a 256 MiB write between launches, the way bench.py flushes between steps).  This is a
development tool: it prints a table and writes gpurun_out/microbench_<tag>.json; it is not a bench line.
B200SEG_LIB selects another build of the library, so two runs give an A/B comparison of two builds on the same box.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pytorchdeeplearing_b200._abi import CudaBackend  # noqa: E402
from pytorchdeeplearing_b200.engine import K3, K1, DOWN, UP  # noqa: E402

DEV = "cuda"


class Timer:
    """Device time per call from CUDA-graph replays (no host launch overhead): INNER calls per graph; the cold
    figure interleaves a 256 MiB write before every call and subtracts a graph holding only the writes."""
    INNER = 10

    def __init__(self, reps, eager=False):
        self.reps = reps
        self.eager = eager
        self.flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
        self.rows = []
        self.flush_us = None

    def _graph(self, body):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            body()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            body()
        torch.cuda.synchronize()
        return g

    def _time(self, g):
        ts = []
        for _ in range(self.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            g.replay()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b) * 1e3)
        ts.sort()
        return ts[len(ts) // 2]

    def run(self, name, fn, bytes_=0, flops=0):
        if self.eager:                 # for ncu: two plain launches per op, no graphs, no timing
            fn()
            fn()
            torch.cuda.synchronize()
            print("ran", name, flush=True)
            return
        if self.flush_us is None:
            def only_flush():
                for _ in range(self.INNER):
                    self.flush.fill_(1)
            self.flush_us = self._time(self._graph(only_flush))

        def warm():
            for _ in range(self.INNER):
                fn()

        def cold():
            for _ in range(self.INNER):
                self.flush.fill_(1)
                fn()
        out = {"warm": self._time(self._graph(warm)) / self.INNER,
               "cold": (self._time(self._graph(cold)) - self.flush_us) / self.INNER}
        row = {"op": name, "warm_us": round(out["warm"], 2), "cold_us": round(out["cold"], 2)}
        if bytes_:
            row["GBps_cold"] = round(bytes_ / out["cold"] / 1e3, 1)
        if flops:
            row["TFLOPs_cold"] = round(flops / out["cold"] / 1e6, 1)
        self.rows.append(row)
        print(f"{name:58s} warm {out['warm']:8.1f} us   cold {out['cold']:8.1f} us"
              + (f"   {row['GBps_cold']:7.1f} GB/s" if bytes_ else "")
              + (f"   {row['TFLOPs_cold']:7.1f} TF/s" if flops else ""), flush=True)


def rnd(shape, dtype=torch.bfloat16, scale=1.0):
    return (torch.randn(shape, device=DEV) * scale).to(dtype)


def bench_stem(be, tm, n, s):
    x = rnd((n, s, s, s, 1), torch.float32)
    for kind, kname, taps in ((K3, "k3", 27), (K1, "k1", 1)):
        w = rnd((16, 1) + ((3, 3, 3) if kind == K3 else (1, 1, 1)), torch.float32, 0.2)
        wp = be.pack_weight(w, kind, "fwd", torch.bfloat16, 3, vox=s ** 3)
        bias = rnd((16,), torch.float32, 0.1)
        y = torch.empty((n, s, s, s, 16), dtype=torch.bfloat16, device=DEV)
        stats = torch.zeros((n, 16, 2), dtype=torch.float64, device=DEV)
        vox = n * s ** 3
        tm.run(f"stem conv[{kname}] 1->16 @{s}^3", lambda: be.conv(kind, 3, x, wp, bias, y, stats, None),
               bytes_=vox * (4 + 32), flops=2 * vox * taps * 16)
        dy = rnd((n, s, s, s, 16))
        dwp = torch.zeros((taps, 1, 16), dtype=torch.float32, device=DEV)
        tm.run(f"stem wgrad[{kname}] 1x16 @{s}^3", lambda: be.wgrad(kind, 3, x, dy, dwp),
               bytes_=vox * (4 + 32), flops=2 * vox * taps * 16)


def bench_stem_gn(be, tm, n, s):
    """the fused input block (csrc/stem_gn.cu): its four launches, beside the nine per-branch launches they replace
    (algorithmic bytes: image 4 B/voxel, 16-channel bf16 tensors 32 B/voxel)"""
    vox = n * s ** 3
    x = rnd((n, s, s, s, 1), torch.float32)
    p3 = be.pack_weight(rnd((16, 1, 3, 3, 3), torch.float32, 0.2), K3, "fwd", torch.bfloat16, 3, vox=s ** 3)
    p1 = be.pack_weight(rnd((16, 1, 1, 1, 1), torch.float32, 0.2), K1, "fwd", torch.bfloat16, 3, vox=s ** 3)
    b3, b1 = rnd((16,), torch.float32, 0.1), rnd((16,), torch.float32, 0.1)
    gamma, beta = rnd((16,), torch.float32) + 1.0, rnd((16,), torch.float32, 0.1)
    st = [torch.zeros((n, 16, 2), dtype=torch.float64, device=DEV) for _ in range(2)]
    be.stem_gn_stats(x, p3, b3, p1, b1, st[0], st[1])
    scale = torch.full((n, 16), 1.25, dtype=torch.float32, device=DEV)
    gn3, gn1 = ((st[i], gamma, beta, scale, s ** 3, 8, 1e-5) for i in range(2))
    cat = torch.empty((n, s, s, s, 32), dtype=torch.bfloat16, device=DEV)
    g = rnd((n, s, s, s, 16))
    sums = [torch.zeros((n, 16, 3), dtype=torch.float64, device=DEV) for _ in range(2)]
    be.stem_gn_bwd_sums(x, p3, b3, p1, b1, gn3, gn1, g, sums[0], sums[1])
    dw3, dw1 = torch.zeros((27, 1, 16), device=DEV), torch.zeros((1, 1, 16), device=DEV)
    d16 = [torch.zeros(16, device=DEV) for _ in range(4)]
    tm.run(f"stem_gn_stats       2x1->16 @{s}^3", lambda: be.stem_gn_stats(x, p3, b3, p1, b1, st[0], st[1]),
           bytes_=vox * 4)
    tm.run(f"stem_gn_apply       2x1->16 @{s}^3", lambda: be.stem_gn_apply(x, p3, b3, p1, b1, gn3, gn1, cat[..., 16:]),
           bytes_=vox * (4 + 32))
    tm.run(f"stem_gn_bwd_sums    2x1->16 @{s}^3",
           lambda: be.stem_gn_bwd_sums(x, p3, b3, p1, b1, gn3, gn1, g, sums[0], sums[1]), bytes_=vox * (4 + 32))
    tm.run(f"stem_gn_bwd         2x1->16 @{s}^3",
           lambda: be.stem_gn_bwd(x, p3, b3, p1, b1, gn3, gn1, g, sums[0], sums[1], dw3, dw1, *d16),
           bytes_=vox * (4 + 32))


def bench_gn(be, tm, n):
    for c, s in ((16, 96), (32, 96), (32, 48), (64, 24), (128, 12), (256, 6)):
        vox = s ** 3
        y = rnd((n, s, s, s, c))
        g = rnd((n, s, s, s, c))
        out = torch.empty_like(y)
        stats = torch.zeros((n, c, 2), dtype=torch.float64, device=DEV)
        yf = y.float()
        stats[:, :, 0] = yf.sum(dim=(1, 2, 3)).double()
        stats[:, :, 1] = (yf * yf).sum(dim=(1, 2, 3)).double()
        gamma, beta = rnd((c,), torch.float32) + 1.0, rnd((c,), torch.float32, 0.1)
        scale = torch.full((n, c), 1.25, dtype=torch.float32, device=DEV)
        gn = (stats, gamma, beta, scale, vox, 8, 1e-5)
        sums = torch.zeros((n, c, 3), dtype=torch.float64, device=DEV)
        dga, dbe, dbi = (torch.zeros(c, dtype=torch.float32, device=DEV) for _ in range(3))
        nb = n * vox * c * 2
        tm.run(f"apply_gn            C={c:3d} @{s}^3", lambda: be.apply_gn(y, gn, None, None, None, out), bytes_=2 * nb)
        tm.run(f"apply_gn(+residual) C={c:3d} @{s}^3", lambda: be.apply_gn(y, gn, None, None, g, out), bytes_=3 * nb)
        tm.run(f"gn_bwd_reduce_gn    C={c:3d} @{s}^3", lambda: be.gn_bwd_reduce_gn(g, y, gn, sums), bytes_=2 * nb)
        tm.run(f"gn_bwd_apply_gn     C={c:3d} @{s}^3",
               lambda: be.gn_bwd_apply_gn(g, y, gn, sums, out, dga, dbe, dbi), bytes_=3 * nb)


def bench_pack(be, tm):
    from pytorchdeeplearing_b200.networks import VNet3d
    m = VNet3d(1, 2).to(DEV)
    reqs, items, nbytes = [], [], 0
    lvl = {16: 96, 32: 48, 64: 24, 128: 12, 256: 6}
    for name, p in m.named_parameters():
        if p.dim() != 5:
            continue
        k = p.shape[2]
        kind = K3 if k == 3 else (K1 if k == 1 else (UP if "up_conv" in name else DOWN))
        if p.shape[1] == 1 or p.shape[0] <= 2:
            continue
        vox = lvl.get(min(p.shape[0], p.shape[1]), 6) ** 3
        for which in ("fwd", "dgrad"):
            reqs.append((p.detach(), kind, which, torch.bfloat16, 3, vox))
            nbytes += p.numel() * 6
        t = p[0, 0].numel()
        items.append((torch.randn((t, p.shape[1], p.shape[0]), device=DEV), torch.empty_like(p)))
    tm.run(f"pack_many  ({len(reqs)} operands)", lambda: be.pack_many(reqs), bytes_=nbytes)
    ub = sum(d.numel() * 8 for d, _ in items)
    tm.run(f"unpack_many ({len(items)} gradients)", lambda: be.unpack_many(items), bytes_=ub)


def bench_wgrad(be, tm, n):
    for (kind, ci, co, s) in ((K3, 16, 16, 96), (K3, 32, 32, 48), (K1, 32, 16, 96), (K3, 64, 64, 24), (K3, 128, 128, 12),
                             (K3, 256, 256, 6)):
        taps = 27 if kind == K3 else 1
        x, dy = rnd((n, s, s, s, ci)), rnd((n, s, s, s, co))
        dwp = torch.zeros((taps, ci, co), dtype=torch.float32, device=DEV)
        vox = n * s ** 3
        tm.run(f"wgrad[k{kind}] {ci}x{co} @{s}^3", lambda: be.wgrad(kind, 3, x, dy, dwp),
               bytes_=vox * (ci + co) * 2, flops=2 * vox * taps * ci * co)


def bench_conv(be, tm, n):
    for (kind, ci, co, s) in ((K3, 16, 16, 96), (K3, 32, 32, 48), (K3, 64, 64, 24), (K3, 128, 128, 12), (K3, 256, 256, 6),
                             (K1, 32, 16, 96), (DOWN, 16, 32, 96), (UP, 32, 16, 48)):
        k = {K3: 3, K1: 1, DOWN: 2, UP: 2}[kind]
        so = s // 2 if kind == DOWN else (s * 2 if kind == UP else s)
        wshape = ((ci, co) if kind == UP else (co, ci)) + (k, k, k)
        w = rnd(wshape, torch.float32, 0.05)
        wp = be.pack_weight(w, kind, "fwd", torch.bfloat16, 3, vox=so ** 3)
        x = rnd((n, s, s, s, ci))
        y = torch.empty((n, so, so, so, co), dtype=torch.bfloat16, device=DEV)
        bias = rnd((co,), torch.float32, 0.1)
        stats = torch.zeros((n, co, 2), dtype=torch.float64, device=DEV)
        vo = n * so ** 3
        taps = k ** 3 if kind != UP else 1
        tm.run(f"conv[k{kind}] {ci}->{co} @{s}^3", lambda: be.conv(kind, 3, x, wp, bias, y, stats, None),
               bytes_=(n * s ** 3 * ci + vo * co) * 2, flops=2 * vo * taps * ci * co)


def bench_convbwd(be, tm, n):
    """data-gradient conv with the GroupNorm-backward sums of the producer layer in its epilogue (b200seg_conv_bwdstats)"""
    for (c, s) in ((32, 48), (64, 24), (128, 12)):
        w = rnd((c, c, 3, 3, 3), torch.float32, 0.05)
        wp = be.pack_weight(w, K3, "dgrad", torch.bfloat16, 3, vox=s ** 3)
        dy, yfwd, add = rnd((n, s, s, s, c)), rnd((n, s, s, s, c)), rnd((n, s, s, s, c))
        g = torch.empty_like(dy)
        yf = yfwd.float()
        stats = torch.stack([yf.sum(dim=(1, 2, 3)).double(), (yf * yf).sum(dim=(1, 2, 3)).double()], -1).contiguous()
        gamma, beta = rnd((c,), torch.float32) + 1.0, rnd((c,), torch.float32, 0.1)
        scale = torch.full((n, c), 1.25, dtype=torch.float32, device=DEV)
        gn = (stats, gamma, beta, scale, s ** 3, 8, 1e-5)
        sums = torch.zeros((n, c, 3), dtype=torch.float64, device=DEV)
        vo = n * s ** 3
        if not be.conv_bwdstats_ok(K3, 3, dy, wp, g, add, yfwd):
            continue
        tm.run(f"conv+gn_bwd_sums {c}->{c} @{s}^3", lambda: be.conv_bwdstats(K3, 3, dy, wp, g, add, yfwd, gn, sums),
               bytes_=vo * c * 2 * 4, flops=2 * vo * 27 * c * c)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--only", default="stem,stemgn,gn,pack,wgrad,conv")
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--tag", default="run")
    ap.add_argument("--eager", action="store_true", help="launch every op twice without graphs/timing (ncu runs)")
    a = ap.parse_args()
    be = CudaBackend()
    tm = Timer(a.reps, a.eager)
    which = set(a.only.split(","))
    with torch.no_grad():
        if "stem" in which:
            bench_stem(be, tm, a.batch, 96)
        if "stemgn" in which:
            bench_stem_gn(be, tm, a.batch, 96)
        if "gn" in which:
            bench_gn(be, tm, a.batch)
        if "pack" in which:
            bench_pack(be, tm)
        if "wgrad" in which:
            bench_wgrad(be, tm, a.batch)
        if "conv" in which:
            bench_conv(be, tm, a.batch)
        if "convbwd" in which:
            bench_convbwd(be, tm, a.batch)
    os.makedirs("gpurun_out", exist_ok=True)
    with open(f"gpurun_out/microbench_{a.tag}.json", "w") as f:
        json.dump({"env": {k: v for k, v in os.environ.items() if k.startswith("B200SEG_")}, "rows": tm.rows}, f, indent=1)


if __name__ == "__main__":
    main()
