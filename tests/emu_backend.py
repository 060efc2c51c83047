"""PyTorch-ops emulation of the C-ABI backend ops -- TEST-ONLY.

A second, independent statement of what every ``b200seg_*`` entry point computes (same
argument meaning as ``pytorchdeeplearing_b200._abi.CudaBackend``).  It lets the CPU suite
validate the host-side layer program and the fused algebra (GroupNorm stats/apply split,
dropout folding, virtual concat, closed-form GroupNorm/loss backward) against the oracle
without a GPU.  The product package never imports this file.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

K3, K1, DOWN, UP = 0, 1, 2, 3


def _ktuple(kind, dims):
    if kind == K3:
        return (3, 3, 3) if dims == 3 else (1, 3, 3)
    if kind == K1:
        return (1, 1, 1)
    return (2, 2, 2) if dims == 3 else (1, 2, 2)


def _ncdhw(t):   # (N,D,H,W,C) view -> (N,C,D,H,W) fp32
    return t.float().permute(0, 4, 1, 2, 3)


def _store(dst, src_ncdhw):
    dst.copy_(src_ncdhw.permute(0, 2, 3, 4, 1).to(dst.dtype))


class EmuBackend:
    name = "emu"

    # ------------------------------------------------------------------ weights
    def pack_weight(self, w, kind, which, dtype, dims, allow_tc=True, vox=None):
        """fwd : gather kinds -> [taps][Cin][Cout] ; UP -> [Cin][taps*Cout]
        dgrad: K3/K1 -> [taps(flipped)][Cout][Cin] ; DOWN -> [Cout][taps*Cin] ; UP -> [taps][Cout][Cin]"""
        a, b = w.shape[0], w.shape[1]
        t = w.numel() // (a * b)
        w3 = w.reshape(a, b, t).float()
        if which == "fwd":
            if kind == UP:       # W (Ci,Co,t) -> [ci][t*Co+co]
                pk = w3.permute(0, 2, 1).reshape(a, t * b)
            else:                # W (Co,Ci,t) -> [t][ci][co]
                pk = w3.permute(2, 1, 0)
        else:
            if kind in (K3, K1):
                pk = w3.flip(2).permute(2, 0, 1)             # [t'][co][ci]
            elif kind == DOWN:   # W (Co,Ci,t) -> [co][t*Ci+ci]
                pk = w3.permute(0, 2, 1).reshape(a, t * b)
            else:                # UP: W (Ci,Co,t) -> [t][co][ci]
                pk = w3.permute(2, 1, 0)
        return pk.contiguous().to(dtype)

    def pack_many(self, reqs):
        return [self.pack_weight(w, kind, which, dtype, dims, vox=vox) for (w, kind, which, dtype, dims, vox) in reqs]

    # plan / launch split of the real backend (engine OV_PACK): the "plan" holds the packed operands, which are only
    # handed to the engine; ``launches`` counts what a real backend would have launched
    def pack_plan(self, reqs):
        import types
        return types.SimpleNamespace(outs=self.pack_many(reqs), launched=False)

    def pack_launch(self, plan, stream=None, after=None):
        assert stream is None and after is None and not plan.launched      # no streams on the CPU
        plan.launched = True
        self.deferred_pack_launches = getattr(self, "deferred_pack_launches", 0) + 1
        return plan.outs

    def unpack_many(self, items):
        for dwp, grad in items:
            grad.copy_(dwp.permute(2, 1, 0).reshape(grad.shape))

    def unpack_wgrad(self, dwp, grad, kind, dims):
        """dwp: gather kinds [t][ci][co] -> grad (Co,Ci,t...) ; UP: [t][co][ci] -> grad (Ci,Co,t...)."""
        grad.copy_(dwp.permute(2, 1, 0).reshape(grad.shape))

    # ------------------------------------------------------------------ conv family
    def conv(self, kind, dims, x, wpk, bias, y, stats, addend):
        k = _ktuple(kind, dims)
        xin = _ncdhw(x)
        wf = wpk.float()
        if kind == UP:
            ci = x.shape[-1]
            t = k[0] * k[1] * k[2]
            co = wf.shape[1] // t
            w = wf.reshape(ci, t, co).permute(0, 2, 1).reshape((ci, co) + k)
            out = F.conv_transpose3d(xin, w, None, stride=k)
        else:
            t, ci, co = wf.shape
            w = wf.permute(2, 1, 0).reshape((co, ci) + k)
            if kind == K3:
                out = F.conv3d(xin, w, None, padding=(k[0] // 2, 1, 1))
            elif kind == K1:
                out = F.conv3d(xin, w, None)
            else:
                out = F.conv3d(xin, w, None, stride=k)
        if bias is not None:
            out = out + bias.float().view(1, -1, 1, 1, 1)
        if stats is not None:
            o64 = out.double()
            stats[..., 0] += o64.sum((2, 3, 4))
            stats[..., 1] += (o64 * o64).sum((2, 3, 4))
        if addend is not None:
            out = out + _ncdhw(addend)
        _store(y, out)

    def conv_bwdstats_ok(self, kind, dims, x, wpk, y, addend, yfwd):
        return kind == K3

    def conv_bwdstats(self, kind, dims, x, wpk, y, addend, yfwd, gn, sums):
        """the data-gradient conv, then the first two backward sums of the layer (yfwd, gn) on the STORED g; sums[..,2]
        (sum of yfwd) is left alone: gn_bwd_apply_gn(sum_y_from_stats=True) takes it from the forward statistics"""
        self.conv(kind, dims, x, wpk, None, y, None, addend)
        tmp = torch.zeros_like(sums)
        self.gn_bwd_reduce_gn(y, yfwd, gn, tmp)
        sums[..., 0:2] += tmp[..., 0:2]

    def wgrad(self, kind, dims, a, b, dwp):
        """dwp[t][ka][kb] += sum_{n,o} a[n, o*s + t - p, ka] * b[n, o, kb]"""
        k = _ktuple(kind, dims)
        A = _ncdhw(a).double()
        B = _ncdhw(b).double()
        s = 2 if kind == DOWN else 1
        pad = (k[0] // 2, k[1] // 2, k[2] // 2) if kind == K3 else (0, 0, 0)
        Ap = F.pad(A, (pad[2], pad[2], pad[1], pad[1], pad[0], pad[0]))
        Do, Ho, Wo = B.shape[2:]
        t = 0
        for kd in range(k[0]):
            for kh in range(k[1]):
                for kw in range(k[2]):
                    sl = Ap[:, :, kd:kd + s * Do:s, kh:kh + s * Ho:s, kw:kw + s * Wo:s]
                    dwp[t] += torch.einsum("nadhw,nbdhw->ab", sl, B).float()
                    t += 1

    # ------------------------------------------------------------------ GroupNorm forward
    def gn_finalize(self, stats, gamma, beta, scale, vox, groups, eps, coef, mr):
        n, c = stats.shape[0], stats.shape[1]
        cpg = c // groups
        m = float(cpg * vox)
        st = stats.view(n, groups, cpg, 2).sum(2)
        mean = st[..., 0] / m
        var = (st[..., 1] / m - mean * mean).clamp_min(0)
        rstd = (var + eps).rsqrt()
        mr[..., 0] = mean.float()
        mr[..., 1] = rstd.float()
        s = scale.double() if scale is not None else torch.ones(n, c, dtype=torch.float64)
        r_c = rstd.repeat_interleave(cpg, 1)
        mu_c = mean.repeat_interleave(cpg, 1)
        g64, b64 = gamma.double(), beta.double()
        coef[..., 0] = (r_c * g64 * s).float()
        coef[..., 1] = ((b64 - mu_c * r_c * g64) * s).float()

    # fused-coefficient forms (composition of the unfused statements above)

    def _coef(self, gn, n, c):
        stats, gamma, beta, scale, vox, groups, eps = gn
        coef, mr = torch.empty(n, c, 2), torch.empty(n, groups, 2)
        self.gn_finalize(stats, gamma, beta, scale, vox, groups, eps, coef, mr)
        return coef, mr

    def apply_gn(self, y1, gn1, y2, gn2, res, out):
        n, c = y1.shape[0], y1.shape[-1]
        c1, _ = self._coef(gn1, n, c)
        c2 = self._coef(gn2, n, c)[0] if y2 is not None else None
        self.apply(y1, c1, y2, c2, res, out)

    def gn_bwd_reduce_gn(self, g, y, gn, sums):
        coef, _ = self._coef(gn, y.shape[0], y.shape[-1])
        self.gn_bwd_reduce(g, y, coef, sums)

    def gn_bwd_apply_gn(self, g, y, gn, sums, dy, dgamma, dbeta, dbias, sum_y_from_stats=False):
        n, c = y.shape[0], y.shape[-1]
        stats, gamma, beta, scale, vox, groups, eps = gn
        if sum_y_from_stats:
            sums = sums.clone()
            sums[..., 2] = stats[..., 0]
        coef, mr = self._coef(gn, n, c)
        coef3 = torch.empty(n, c, 3)
        dbi = torch.zeros_like(dbias) if dbias is not None else None      # the fused form ACCUMULATES the bias gradient
        self.gn_bwd_finalize(sums, mr, gamma, scale, vox, groups, coef3, dgamma, dbeta, dbi)
        if dbias is not None:
            dbias += dbi
        self.gn_bwd_apply(g, y, coef, coef3, dy)

    def apply(self, y1, c1, y2, c2, res, out):
        def one(y, c):
            a = c[..., 0].view(c.shape[0], 1, 1, 1, -1)
            b = c[..., 1].view(c.shape[0], 1, 1, 1, -1)
            return torch.relu(torch.addcmul(b, y.float(), a))
        v = one(y1, c1)
        if y2 is not None:
            v = v + one(y2, c2)
        if res is not None:
            v = v + res.float()
        out.copy_(v.to(out.dtype))

    # ------------------------------------------------------------------ pooling
    def pool_fwd(self, x, out, dims):
        k = (2, 2, 2) if dims == 3 else (1, 2, 2)
        _store(out, F.max_pool3d(_ncdhw(x), k, k))

    def pool_bwd(self, x, g_out, addend, g_x, dims):
        k = (2, 2, 2) if dims == 3 else (1, 2, 2)
        with torch.enable_grad():
            xin = _ncdhw(x).detach().requires_grad_(True)
            o = F.max_pool3d(xin, k, k)
            (gx,) = torch.autograd.grad(o, xin, _ncdhw(g_out))
        if addend is not None:
            gx = gx + _ncdhw(addend)
        _store(g_x, gx)

    # ------------------------------------------------------------------ GroupNorm backward
    def gn_bwd_reduce(self, g, y, coef, sums):
        n = y.shape[0]
        a = coef[..., 0].view(n, 1, 1, 1, -1)
        b = coef[..., 1].view(n, 1, 1, 1, -1)
        yf = y.float()
        mask = torch.addcmul(b, yf, a) > 0
        d0 = (g.float() * mask).double()
        sums[..., 0] += d0.sum((1, 2, 3))
        sums[..., 1] += (d0 * yf.double()).sum((1, 2, 3))
        sums[..., 2] += yf.double().sum((1, 2, 3))

    def gn_bwd_finalize(self, sums, mr, gamma, scale, vox, groups, coef3, dgamma, dbeta, dbias):
        n, c = sums.shape[0], sums.shape[1]
        cpg = c // groups
        m = float(cpg * vox)
        s = scale.double() if scale is not None else torch.ones(n, c, dtype=torch.float64)
        mu = mr[..., 0].double().repeat_interleave(cpg, 1)
        r = mr[..., 1].double().repeat_interleave(cpg, 1)
        g64 = gamma.double()
        s1 = sums[..., 0] * s
        s2 = sums[..., 1] * s
        s3 = sums[..., 2]
        dbeta += s1.sum(0).float()
        dgamma += (r * (s2 - mu * s1)).sum(0).float()
        sa = (g64 * s1).view(n, groups, cpg).sum(2).repeat_interleave(cpg, 1)
        sax = (g64 * r * (s2 - mu * s1)).view(n, groups, cpg).sum(2).repeat_interleave(cpg, 1)
        m1, m2 = sa / m, sax / m
        p = r * g64 * s
        q = -r * r * m2
        rr = -r * m1 + r * r * mu * m2
        coef3[..., 0] = p.float()
        coef3[..., 1] = q.float()
        coef3[..., 2] = rr.float()
        if dbias is not None:
            dbias.copy_((r * g64 * s1 + q * s3 + rr * vox).sum(0).float())

    def gn_bwd_apply(self, g, y, coef, coef3, dy):
        n = y.shape[0]
        v = lambda t, i: t[..., i].view(n, 1, 1, 1, -1)
        yf = y.float()
        mask = torch.addcmul(v(coef, 1), yf, v(coef, 0)) > 0
        out = g.float() * mask * v(coef3, 0) + yf * v(coef3, 1) + v(coef3, 2)
        dy.copy_(out.to(dy.dtype))

    def colsum(self, dy, out):
        out += dy.double().sum((0, 1, 2, 3)).float()

    # ------------------------------------------------------------------ trilinear 2x upsample + skip add (UNet3dthin)
    def upsample_add(self, a, e, s):
        up = F.interpolate(_ncdhw(a), scale_factor=(2, 2, 2), mode="trilinear")
        _store(s, up + _ncdhw(e))

    def upsample_bwd(self, g_s, g_a):
        with torch.enable_grad():
            a = torch.zeros(_ncdhw(g_a).shape, requires_grad=True)
            up = F.interpolate(a, scale_factor=(2, 2, 2), mode="trilinear")
            (ga,) = torch.autograd.grad(up, a, _ncdhw(g_s))
        _store(g_a, ga)

    # ------------------------------------------------------------------ classifier head (ResNet2d / ResNet3d)
    def cls_head_fwd(self, x, w1, b1, w2, b2, pooled, hidden, logits):
        p = x.float().reshape(x.shape[0], -1, x.shape[-1]).mean(1)
        h = F.relu(F.linear(p, w1, b1))
        pooled.copy_(p)
        hidden.copy_(h)
        logits.copy_(F.linear(h, w2, b2))

    def cls_head_bwd(self, dlogits, pooled, hidden, w1, w2, work, dx, dw1, db1, dw2, db2):
        n, c = pooled.shape
        vox = dx.numel() // (n * c)
        dh = (dlogits @ w2) * (hidden > 0)
        dp = (dh @ w1) / vox
        dw1.copy_(dh.t() @ pooled)
        db1.copy_(dh.sum(0))
        dw2.copy_(dlogits.t() @ hidden)
        db2.copy_(dlogits.sum(0))
        dx.copy_(dp.view(n, 1, 1, 1, c).expand(dx.shape).to(dx.dtype))

    # ------------------------------------------------------------------ head + losses
    def head_probs(self, logits, probs):
        if logits.shape[-1] == 1:
            probs.copy_(torch.sigmoid(logits))
        else:
            probs.copy_(torch.softmax(logits, dim=-1))

    def head_fwd(self, x, w, bias, logits, probs):
        nc = logits.shape[-1]
        if nc > 8 or x.shape[-1] % 4 != 0:
            return False
        z = torch.einsum("ndhwk,ck->ndhwc", x.float(), w.reshape(nc, -1).float())
        if bias is not None:
            z = z + bias.float()
        logits.copy_(z)
        if probs is not None:
            self.head_probs(logits, probs)
        return True

    def head_bwd(self, x, dlogits, w, dx, dw, db):
        nc, cin = dlogits.shape[-1], x.shape[-1]
        if nc > 4 or cin not in (16, 32):
            return False
        w2 = w.reshape(nc, cin).double()
        g = dlogits.double()
        dx.copy_(torch.einsum("ndhwc,ck->ndhwk", g, w2).to(dx.dtype))
        dw += torch.einsum("ndhwc,ndhwk->ck", g, x.double()).reshape(dw.shape).float()
        db += g.sum((0, 1, 2, 3)).float()
        return True

    @staticmethod
    def part_size(c):
        return 3 * c + 4 if c > 1 else 7

    def loss_partials(self, logits, labels, gamma, alpha_f, part, metric=None):
        """part (double): multi-class C>1: [I_c]*C, [P_c]*C, [Cnt_c]*C, sum_nll, sum_focal, V, BAD
                          binary  C==1: I, P, T, sum_bce, sum_focal(alpha folded), V, BAD
        metric (double [N][C][3], optional): per sample/class {sum [p>.5][t==c], sum [p>.5], sum [t==c]}"""
        c = logits.shape[-1]
        n = logits.shape[0]
        z = logits.reshape(-1, c).double()
        t = labels.reshape(-1)
        if c == 1:
            zf, tf = z[:, 0], t.double()
            p = torch.sigmoid(zf)
            b = zf.clamp_min(0) - zf * tf + torch.log1p(torch.exp(-zf.abs()))
            pt = torch.exp(-b)
            vals = [(p * tf).sum(), p.sum(), tf.sum(), b.sum(), (alpha_f * (1 - pt) ** gamma * b).sum(),
                    torch.tensor(float(zf.numel()), dtype=torch.float64)]
            part[:6] += torch.stack(vals)
            if metric is not None:
                on = (torch.sigmoid(logits.reshape(n, -1).float()) > 0.5).double()
                tn = labels.reshape(n, -1).double()
                metric[:, 0, 0] += (on * tn).sum(1)
                metric[:, 0, 1] += on.sum(1)
                metric[:, 0, 2] += tn.sum(1)
        else:
            bad = (t < 0) | (t >= c)
            part[3 * c + 3] += float(bad.sum())
            keep = ~bad
            z, tk = z[keep], t[keep]
            p = torch.softmax(z, 1)
            oh = F.one_hot(tk.long(), c).double()
            logp = torch.log_softmax(z, 1)
            nll = -(logp * oh).sum(1)
            ptt = torch.exp(-nll)
            part[0:c] += (p * oh).sum(0)
            part[c:2 * c] += p.sum(0)
            part[2 * c:3 * c] += oh.sum(0)
            part[3 * c] += nll.sum()
            part[3 * c + 1] += ((1 - ptt) ** gamma * nll).sum()
            part[3 * c + 2] += float(t.shape[0])
            if metric is not None:
                on = (torch.softmax(logits.reshape(n, -1, c).float(), -1) > 0.5).double()
                ohn = F.one_hot(labels.reshape(n, -1).long().clamp(0, c - 1), c).double()
                metric[..., 0] += (on * ohn).sum(1)
                metric[..., 1] += on.sum(1)
                metric[..., 2] += ohn.sum(1)

    def metric_partials(self, probs, labels, threshold, metric):
        n, c = probs.shape[0], probs.shape[-1]
        on = (probs.reshape(n, -1, c) > threshold).double()
        if c == 1:
            tn = labels.reshape(n, -1, 1).double()
        else:
            tn = F.one_hot(labels.reshape(n, -1).long(), c).double()
        metric[..., 0] += (on * tn).sum(1)
        metric[..., 1] += on.sum(1)
        metric[..., 2] += tn.sum(1)

    def metric_finalize(self, metric, out):
        n, c = metric.shape[0], metric.shape[1]
        s = 1e-5
        cls = [0] if c == 1 else list(range(1, c))
        m = metric[:, cls]
        dice = ((2 * m[..., 0] + s) / (m[..., 1] + m[..., 2] + s)).mean(0).mean()
        iou = ((m[..., 0] + s) / (m[..., 1] + m[..., 2] - m[..., 0] + s)).mean(0).mean()
        out[0], out[1] = dice.float(), iou.float()

    def head_mask(self, x, w, bias, mask, threshold):
        nc = w.shape[0]
        if nc > 8 or x.shape[-1] % 4 != 0:
            return False
        z = torch.einsum("ndhwk,ck->ndhwc", x.float(), w.reshape(nc, -1).float())
        if bias is not None:
            z = z + bias.float()
        self.mask_logits(z, threshold, mask)
        return True

    def stage_images_u8(self, img, out):
        a = img.double()
        dims = tuple(range(1, a.dim()))
        mean = a.mean(dims, keepdim=True)
        sd = ((a - mean) ** 2).mean(dims, keepdim=True).sqrt()
        out.copy_(((a - mean) / sd).float().reshape(out.shape).to(out.dtype))
        return out

    def stage_labels_u8(self, lab, out, binarize=True):
        out.copy_(((lab != 0).long() if binarize else lab.long()).reshape(out.shape))
        return out

    def mask_logits(self, logits, threshold, mask):
        if logits.shape[-1] == 1:
            mask.copy_(((torch.sigmoid(logits[..., 0]) > threshold) * 255).to(torch.uint8).reshape(mask.shape))
        else:
            mask.copy_(logits.argmax(-1).to(torch.uint8).reshape(mask.shape))

    def adam_step(self, param, grad, exp_avg, exp_avg_sq, state, lr, beta1, beta2, eps, weight_decay, decoupled,
                  gscale=None, tick=True):
        if tick:
            state[0] += 1
            t = float(state[0])
            state[1] = lr / (1 - beta1 ** t)
            state[2] = (1 - beta2 ** t) ** 0.5
        g = grad * (gscale if gscale is not None else 1.0)
        if decoupled:
            param.mul_(1 - lr * weight_decay)
        else:
            g = g + weight_decay * param
        exp_avg.lerp_(g, 1 - beta1)
        exp_avg_sq.mul_(beta2).addcmul_(g, g, value=1 - beta2)
        denom = (exp_avg_sq.sqrt() / state[2]).add_(eps)
        param.addcdiv_(exp_avg, denom, value=-float(state[1]))

    def loss_finalize(self, part, c, terms, alpha, gamma, alpha_f, loss, lcoef):
        """terms bitmask: 1 dice, 2 ce/bce, 4 focal.  lcoef (fp32):
        multi : a_c (C), b_c (C), ce_scale, focal_scale, gamma
        binary: a, b, bce_scale, focal_scale(alpha folded), gamma"""
        s, eps = 1e-5, 1e-7
        pt = part.double()
        if c == 1:
            I, P, T, sb, sf, V = [pt[i] for i in range(6)]
            val = torch.zeros((), dtype=torch.float64)
            a = b = torch.zeros((), dtype=torch.float64)
            den = P + T + s
            if terms & 1:
                val = val + 1.0 - (2 * I + s) / den.clamp_min(eps)
                a, b = -2.0 / den, (2 * I + s) / (den * den)
            if terms & 2:
                val = val + sb / V
            if terms & 4:
                val = val + sf / V
            lcoef[0], lcoef[1] = a.float(), b.float()
            lcoef[2] = (1.0 / V).float() if terms & 2 else 0.0
            lcoef[3] = (alpha_f / V).float() if terms & 4 else 0.0
            lcoef[4] = float(gamma)
        else:
            I, Ps, Cn = pt[0:c], pt[c:2 * c], pt[2 * c:3 * c]
            snll, sfoc, V = pt[3 * c], pt[3 * c + 1], pt[3 * c + 2]
            present = (Cn > 0).double()
            K = present.sum()
            val = torch.zeros((), dtype=torch.float64)
            a = torch.zeros(c, dtype=torch.float64)
            b = torch.zeros(c, dtype=torch.float64)
            if terms & 1:
                D = Cn + Ps
                d_raw = (2 * I + s) / (D + s)
                d = d_raw.clamp_min(eps)
                al = alpha.double()
                val = val + (-(d * present * al)).sum() / K
                w = al * present / K * (d_raw >= eps).double()
                a = -2.0 * w / (D + s)
                b = w * (2 * I + s) / ((D + s) ** 2)
            if terms & 2:
                val = val + snll / V
            if terms & 4:
                val = val + sfoc / V
            lcoef[0:c] = a.float()
            lcoef[c:2 * c] = b.float()
            lcoef[2 * c] = (1.0 / V).float() if terms & 2 else 0.0
            lcoef[2 * c + 1] = (1.0 / V).float() if terms & 4 else 0.0
            lcoef[2 * c + 2] = float(gamma)
            if pt[3 * c + 3] > 0:
                val = val * float("nan")
        loss.copy_(val.float())

    def loss_bwd(self, logits, labels, lcoef, gscale, dlogits):
        c = logits.shape[-1]
        z = logits.reshape(-1, c).double()
        t = labels.reshape(-1)
        lc = lcoef.double()
        if c == 1:
            zf, tf = z[:, 0], t.double()
            p = torch.sigmoid(zf)
            a, b, cs, fs, gamma = [lc[i] for i in range(5)]
            bce = zf.clamp_min(0) - zf * tf + torch.log1p(torch.exp(-zf.abs()))
            pt = torch.exp(-bce)
            g = (tf * a + b) * p * (1 - p) + cs * (p - tf)
            g = g + fs * ((1 - pt) ** gamma + gamma * (1 - pt) ** (gamma - 1) * pt * bce) * (p - tf)
            out = g.unsqueeze(1)
        else:
            a, b = lc[0:c], lc[c:2 * c]
            cs, fs, gamma = lc[2 * c], lc[2 * c + 1], lc[2 * c + 2]
            p = torch.softmax(z, 1)
            oh = F.one_hot(t.long(), c).double()
            gd = oh * a + b
            out = p * (gd - (gd * p).sum(1, keepdim=True))
            nll = -(torch.log_softmax(z, 1) * oh).sum(1, keepdim=True)
            ptt = torch.exp(-nll)
            out = out + cs * (p - oh)
            out = out + fs * ((1 - ptt) ** gamma + gamma * (1 - ptt) ** (gamma - 1) * ptt * nll) * (p - oh)
        dlogits.copy_((out * gscale.double()).float().reshape(dlogits.shape))
