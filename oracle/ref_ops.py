"""TEST INFRASTRUCTURE — plain-torch reference of every device op behind pydreamer_b200.ops.NativeOps.

Same method names and argument meaning as NativeOps, written with stock torch ops (works on CPU
and CUDA, fp32 or fp64).  It is the checker for (a) each hand-written kernel (tests/test_kernels_gpu.py
compares NativeOps against this on the same inputs) and (b) the host-side composition + hand-written
backward of pydreamer_b200.dreamer (tests/test_dreamer_cpu.py runs the module on this table on CPU and
compares with the reference implementation's autograd).  Only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline leg may import it; the product path never does.

Reference lines each op restates are the ones cited in include/pd_b200.h.

Each method refuses (RuntimeError) the arguments its native entry point refuses with PD_REQUIRE: leading dimensions,
16-byte alignment, the smallest tensor-core shapes and the row / class / channel / horizon limits of the kernels.  A
schedule that runs on this table therefore also passes the native host checks.  The persistent-kernel stand-ins take the
shapes their kernels take on a 148-SM GPU (SMS).
"""
import math

import torch
import torch.nn.functional as F

ACT_NONE, ACT_ELU = 0, 1
SMS = 148                   # SM count the persistent RSSM stand-ins assume (Dreamer's predicates do the same off the GPU)


def _require(cond, what):
    """PD_REQUIRE of the native entry point: the same condition refuses the call here."""
    if not cond:
        raise RuntimeError(f"{what} unsupported")


def _ld(t):
    """Row stride (elements) of a 2-D view, as NativeOps passes it."""
    return t.stride(0) if t.shape[0] > 1 else max(t.stride(0), t.shape[1])


def _aligned(t, n=16):
    return t is None or t.data_ptr() % n == 0


def _cdiv(a, b):
    return -(-a // b)


def _act(x, act):
    return F.elu(x) if act == ACT_ELU else x


def _elu_grad_from_out(y):
    return torch.where(y > 0, torch.ones_like(y), y + 1)


def _group_softmax(logits, G, C):
    l = logits.reshape(logits.shape[0], G, C)
    ln = l - l.logsumexp(-1, keepdim=True)
    return ln, F.softmax(ln, -1)


class RefOps:
    is_reference = True

    def __init__(self, device="cpu"):
        self.device = torch.device(device)
        self._launches = 0

    def set_gemm_impl(self, impl):
        pass

    def set_round_operands(self, on):
        pass

    def launch_count(self):
        return self._launches

    # ------------------------------------------------------------------ gemm
    def gemm(self, A, B, C, *, a_mn=False, b_mn=False, bias=None, res=None, r_div=1, act=ACT_NONE,
             round_out=False, accumulate=False, c_zeroed=False):
        _require(C.numel() > 0 and (A.shape[0] if a_mn else A.shape[1]) > 0, f"pd_gemm: shape {tuple(C.shape)}")
        _require(not (accumulate and (bias is not None or res is not None or act != ACT_NONE)),
                 "pd_gemm: accumulate with bias / residual / activation")
        _require(not (C.dtype == torch.float16 and (accumulate or res is not None)),
                 "pd_gemm: an fp16 output accumulating or adding a residual")
        a = A.t() if a_mn else A
        b = B if b_mn else B.t()
        v = a @ b
        if accumulate:
            C.add_(v)
            return C
        if bias is not None:
            v = v + bias
        if res is not None:
            rows = torch.arange(C.shape[0], device=C.device) // r_div
            v = v + res[rows]
        C.copy_(_act(v, act))
        return C

    # ------------------------------------------------------------------ rowwise
    def gemm_f16(self, A16, B16, C, *, bias=None, res=None, r_div=1, act=ACT_NONE, round_out=False):
        (M, N), K = C.shape, A16.shape[1]
        _require(M > 0 and N >= 8 and K >= 8, f"pd_gemm_f16: shape {M} {N} {K}")
        _require(_ld(A16) % 8 == 0 and _ld(B16) % 8 == 0, f"pd_gemm_f16: lda {_ld(A16)} ldb {_ld(B16)} (% 8)")
        _require(_aligned(A16) and _aligned(B16), "pd_gemm_f16: operands not 16-byte aligned")
        return self.gemm(A16.to(C.dtype), B16.to(C.dtype), C, bias=bias, res=res, r_div=r_div, act=act)

    def conv_gemm(self, mode, X, k, O, Cmat, *, o_mn=False, bias=None, act=ACT_NONE, round_out=False):
        NB, H, W, C = X.shape
        _require(mode in (1, 2, 3), f"pd_conv_gemm: mode {mode}")
        _require(C % 4 == 0 and _aligned(X), f"pd_conv_gemm: C={C} (% 4) / X alignment")
        _require(_ld(O) % 4 == 0 and _aligned(O), f"pd_conv_gemm: ldo={_ld(O)} (% 4) / operand alignment")
        _require(_ld(Cmat) % 4 == 0 and _aligned(Cmat), f"pd_conv_gemm: ldc={_ld(Cmat)} (% 4) / output alignment")
        P, Q = (H - k) // 2 + 1, (W - k) // 2 + 1
        pat = X.unfold(1, k, 2).unfold(2, k, 2).permute(0, 1, 2, 4, 5, 3).reshape(NB * P * Q, k * k, C)   # (pixels, tap, c)
        if mode == 1:
            v = pat.reshape(NB * P * Q, k * k * C) @ (O if o_mn else O.t())
            if bias is not None:
                v = v + bias
            Cmat.copy_(_act(v, act))
            return Cmat
        cpad = (C + 31) // 32 * 32
        colp = torch.zeros(NB * P * Q, k * k, cpad, dtype=X.dtype, device=X.device)
        colp[:, :, :C] = pat
        colp = colp.reshape(NB * P * Q, k * k * cpad)
        if mode == 2:
            Cmat.add_(colp.t() @ O)
        else:
            Cmat.add_(O.t() @ colp)
        return Cmat

    def to_half(self, src, dst):
        dst.copy_(src.to(dst.dtype))

    def ln_elu_fwd(self, x, gamma, beta, eps, y, mean, rstd, y16=None):
        _require(1 <= x.shape[1] <= 1024, f"pd_ln_elu_fwd: N={x.shape[1]} (1..1024)")
        mu = x.mean(-1)
        var = x.var(-1, unbiased=False)
        r = 1.0 / torch.sqrt(var + eps)
        mean.copy_(mu)
        rstd.copy_(r)
        y.copy_(F.elu((x - mu[:, None]) * r[:, None] * gamma + beta))
        if y16 is not None:
            y16.copy_(y.to(y16.dtype))

    def ln_elu_bwd(self, dy, x, y, gamma, mean, rstd, dx, dgamma, dbeta, dbias=None):
        _require(1 <= x.shape[1] <= 1024, f"pd_ln_elu_bwd: N={x.shape[1]} (1..1024)")
        g = dy * _elu_grad_from_out(y)
        xh = (x - mean[:, None]) * rstd[:, None]
        dgamma.add_((g * xh).sum(0))
        dbeta.add_(g.sum(0))
        dxh = g * gamma
        c1 = dxh.mean(-1, keepdim=True)
        c2 = (dxh * xh).mean(-1, keepdim=True)
        d = rstd[:, None] * (dxh - c1 - xh * c2)
        if dbias is not None:
            dbias.add_(d.sum(0))
        dx.copy_(d)

    def gru_fwd(self, gi, gh, hprev, hout, hmask=None, mask_next=None, gates=None, h16=None):
        D = hprev.shape[1]
        r = torch.sigmoid(gi[:, :D] + gh[:, :D])
        u = torch.sigmoid(gi[:, D:2 * D] + gh[:, D:2 * D])
        ghn = gh[:, 2 * D:3 * D]
        n = torch.tanh(gi[:, 2 * D:3 * D] + r * ghn)
        hn = (1 - u) * n + u * hprev
        if gates is not None:
            gates.view(-1, 4, D).copy_(torch.stack([r, u, n, ghn], 1))
        hout.copy_(hn)
        if h16 is not None:
            h16.copy_(hn.to(h16.dtype))
        if hmask is not None:
            hmask.copy_(hn * mask_next[:, None])

    def gru_bwd(self, dh_a, dh_b, mask_b, gates, hprev, dgi, dgh, dh_carry):
        D = hprev.shape[1]
        dh = torch.zeros_like(hprev)
        if dh_a is not None:
            dh = dh + dh_a
        if dh_b is not None:
            dh = dh + (dh_b * mask_b[:, None] if mask_b is not None else dh_b)
        g = gates.view(-1, 4, D)
        r, u, n, ghn = g[:, 0], g[:, 1], g[:, 2], g[:, 3]
        dn_pre = dh * (1 - u) * (1 - n * n)
        du_pre = dh * (hprev - n) * u * (1 - u)
        dr_pre = dn_pre * ghn * r * (1 - r)
        dgi.copy_(torch.cat([dr_pre, du_pre, dn_pre], 1))
        dgh.copy_(torch.cat([dr_pre, du_pre, dn_pre * r], 1))
        dh_carry.copy_(dh * u)

    def rssm_unroll_fwd(self, dims, eps, **t):
        """Torch statement of pd_rssm_unroll_fwd (csrc/pd_rssm_fwd3.cu; rssm.py:21-78, 125-153): the whole posterior
        unroll in one call, fp16 weights, LayerNorm outputs and h rounded to fp16 (they are the tensor-core operands)."""
        T, BI, I, D, Hd, G, C = (int(dims[k]) for k in ("T", "BI", "I", "D", "Hd", "G", "C"))
        RG = SMS // (4 if D % 256 == 0 else 1)
        _require(T >= 1 and 1 <= BI <= 256 and I >= 1 and BI % I == 0 and Hd <= 1024 and Hd % 8 == 0 and D % 8 == 0 and
                 1 <= C <= 32 and 1 <= G <= min(SMS, 256) and _cdiv(D, SMS) <= 16 and _cdiv(D, RG) <= 64 and
                 _cdiv(Hd, RG) <= 32, f"pd_rssm_unroll_fwd: shape {dict(dims)}")
        B = BI // I
        x1, za, m1, r1, gates, feat, hin, zin = (t[k] for k in ("x1", "za", "m1", "r1", "gates", "feat", "hin", "zin"))
        y2, pin, m2, r2, post, idx = (t[k] for k in ("y2", "pin", "m2", "r2", "post", "idx"))
        aa, ea, mask, noise = t["aa"], t.get("ea"), t["mask"], t["noise"]
        dt = x1.dtype
        Wz, Wih, Whh, Wph, Wpm = (t[k].to(dt) for k in ("w_z16", "w_ih16", "w_hh16", "w_ph16", "w_pm16"))
        h16 = lambda v: v.to(torch.float16).to(dt)
        rep = lambda v: v.repeat_interleave(I, 0) if I > 1 else v

        def ln(x, g, b):
            mu, var = x.mean(-1), x.var(-1, unbiased=False)
            r = 1.0 / torch.sqrt(var + eps)
            return h16(F.elu((x - mu[:, None]) * r[:, None] * g + b)), mu, r

        gh = h16(hin[0]) @ Whh.t()                                       # raw product; mask and bias applied at use
        for s in range(T):
            m = mask[s] if s > 0 else torch.ones_like(mask[0])           # h_0 / z_0 arrive masked
            if s > 0:
                zprev = feat[s - 1][:, D:]
                x1[s].copy_(m[:, None] * (zprev @ Wz.t()) + t["b_z"] + rep(aa[s * B:(s + 1) * B]))
                zin[s].copy_(zprev * m[:, None])
            y, mu, r = ln(x1[s], t["ln1_g"], t["ln1_b"])
            za[s].copy_(y); m1[s].copy_(mu); r1[s].copy_(r)
            gi = y @ Wih.t() + t["b_ih"]
            ghb = m[:, None] * gh + t["b_hh"]
            rg = torch.sigmoid(gi[:, :D] + ghb[:, :D])
            ug = torch.sigmoid(gi[:, D:2 * D] + ghb[:, D:2 * D])
            ghn = ghb[:, 2 * D:]
            ng = torch.tanh(gi[:, 2 * D:] + rg * ghn)
            hn = h16((1 - ug) * ng + ug * hin[s])
            feat[s][:, :D].copy_(hn)
            gates[s].view(BI, 4, D).copy_(torch.stack([rg, ug, ng, ghn], 1))
            if s + 1 < T:
                hin[s + 1].copy_(hn * mask[s + 1][:, None])
            v = hn @ Wph.t() + t["b_ph"]
            if ea is not None:
                v = v + rep(ea[s * B:(s + 1) * B])
            y2[s].copy_(v)
            gh = hn @ Whh.t()
            y, mu, r = ln(y2[s], t["ln2_g"], t["ln2_b"])
            pin[s].copy_(y); m2[s].copy_(mu); r2[s].copy_(r)
            post[s].copy_(y @ Wpm.t() + t["b_pm"])
            _, p = _group_softmax(post[s], G, C)
            k = (p / noise[s].reshape(BI, G, C)).argmax(-1)
            idx[s].copy_(k.to(idx.dtype))
            feat[s][:, D:].copy_(F.one_hot(k, C).to(dt).reshape(BI, G * C))

    def transpose_to_half(self, src, dst):
        dst.copy_(src.t().to(dst.dtype))

    def rssm_unroll_bwd(self, dims, kl_weight, round_out=True, **t):
        """Torch statement of pd_rssm_unroll_bwd (csrc/pd_rssm_bptt.cu): BPTT of the posterior unroll for all T steps,
        transposed fp16 weights, same per-step formulas as the chain cat_st_bwd / ln_elu_bwd / gru_bwd of this table."""
        T, BI, D, Hd, G, C = (int(dims[k]) for k in ("T", "BI", "D", "Hd", "G", "C"))
        Z = G * C
        RG2, RG6 = SMS // (4 if Z % 256 == 0 else 1), SMS // (4 if (3 * D) % 256 == 0 else 1)
        R = max(1, min(4, SMS // G))
        _require(T >= 1 and 1 <= BI <= min(64, SMS) and Hd <= 1024 and Hd % 8 == 0 and D % 8 == 0 and Z % 8 == 0 and
                 1 <= C <= 32 and 1 <= G <= SMS and _cdiv(BI, R) <= 16 and _cdiv(D, SMS) <= 16 and _cdiv(Hd, RG2) <= 32 and
                 _cdiv(D, RG6) <= 64 and _cdiv(Hd, RG6) <= 32, f"pd_rssm_unroll_bwd: shape {dict(dims)}")
        dt = t["dpost"].dtype
        WpmT, WphT, WhhT, WihT, WzT = (t[k].to(dt) for k in ("w_pmT16", "w_phT16", "w_hhT16", "w_ihT16", "w_zT16"))
        v3 = lambda k, n: t[k].view(T, BI, n)
        post, pin, y2, x1, za = v3("post", Z), v3("pin", Hd), v3("y2", Hd), v3("x1", Hd), v3("za", Hd)
        gates, hin, dfeat, dpu = v3("gates", 4 * D), v3("hin", D), v3("dfeat", D + Z), v3("dpost_u", Z)
        m2, r2, m1, r1, mask, w = (t[k].view(T, BI) for k in ("m2", "r2", "m1", "r1", "mask", "w"))
        dpost, dy2, dgi, dgh, dx1 = v3("dpost", Z), v3("dy2", Hd), v3("dgi", 3 * D), v3("dgh", 3 * D), v3("dx1", Hd)

        def ln_bwd(dy, x, y, gamma, mean, rstd, gg, gb, gx):
            g_ = dy * _elu_grad_from_out(y)
            xh = (x - mean[:, None]) * rstd[:, None]
            dxh = g_ * gamma
            c1, c2 = dxh.mean(-1, keepdim=True), (dxh * xh).mean(-1, keepdim=True)
            d = rstd[:, None] * (dxh - c1 - xh * c2)
            gg.add_((g_ * xh).sum(0)); gb.add_(g_.sum(0)); gx.add_(d.sum(0))
            return d

        dzin_next = dhin_next = None
        for s in reversed(range(T)):
            nxt = s + 1 < T
            dz = dfeat[s][:, D:].clone()
            if nxt:
                dz = dz + dzin_next * mask[s + 1][:, None]
            _, p = _group_softmax(post[s], G, C)
            dzg = dz.view(BI, G, C)
            dp = (p * (dzg - (p * dzg).sum(-1, keepdim=True))).reshape(BI, Z) + kl_weight * w[s][:, None] * dpu[s]
            dpost[s].copy_(dp)
            dpin = dpost[s] @ WpmT.t()
            dy2[s].copy_(ln_bwd(dpin, y2[s], pin[s], t["ln2_g"], m2[s], r2[s], t["g_ln2_g"], t["g_ln2_b"], t["g_b_ph"]))
            dh = dy2[s] @ WphT.t() + dfeat[s][:, :D]
            if nxt:
                dh = dh + dhin_next * mask[s + 1][:, None]
            gt = gates[s].view(BI, 4, D)
            rg, ug, ng, ghn = gt[:, 0], gt[:, 1], gt[:, 2], gt[:, 3]
            dn = dh * (1 - ug) * (1 - ng * ng)
            du = dh * (hin[s] - ng) * ug * (1 - ug)
            dr = dn * ghn * rg * (1 - rg)
            dgi[s].copy_(torch.cat([dr, du, dn], 1))
            dgh[s].copy_(torch.cat([dr, du, dn * rg], 1))
            dhin_next = dgh[s] @ WhhT.t() + dh * ug
            dza = dgi[s] @ WihT.t()
            dx1[s].copy_(ln_bwd(dza, x1[s], za[s], t["ln1_g"], m1[s], r1[s], t["g_ln1_g"], t["g_ln1_b"], t["g_b_z"]))
            dzin_next = dx1[s] @ WzT.t()

    def cat_sample(self, logits, noise, G, C, z, zmask=None, mask_next=None, idx=None, z16=None):
        _require(1 <= C <= 32, f"pd_cat_sample: C={C} (<= 32)")
        M = logits.shape[0]
        _, p = _group_softmax(logits, G, C)
        k = (p / noise.reshape(M, G, C)).argmax(-1)
        zz = F.one_hot(k, C).to(logits.dtype).reshape(M, G * C)
        z.copy_(zz)
        if z16 is not None:
            z16.copy_(zz.to(z16.dtype))
        if zmask is not None:
            zmask.copy_(zz * mask_next[:, None])
        if idx is not None:
            idx.copy_(k.to(idx.dtype))

    def cat_st_bwd(self, logits, G, C, dz_a, dz_b, mask_b, extra, rowscale, alpha, dlogits):
        _require(1 <= C <= 32, f"pd_cat_st_bwd: C={C} (<= 32)")
        M = logits.shape[0]
        _, p = _group_softmax(logits, G, C)
        dz = torch.zeros(M, G * C, dtype=logits.dtype, device=logits.device)
        if dz_a is not None:
            dz = dz + dz_a
        if dz_b is not None:
            dz = dz + (dz_b * mask_b[:, None] if mask_b is not None else dz_b)
        dz = dz.reshape(M, G, C)
        d = (p * (dz - (p * dz).sum(-1, keepdim=True))).reshape(M, G * C)
        if extra is not None:
            sc = rowscale[:, None] if rowscale is not None else 1.0
            d = d + alpha * sc * extra
        dlogits.copy_(d)

    def kl(self, post, prior, idx, mode, balance, G, C, loss_kl, kl_exact, ent_post, ent_prior, dpost, dprior):
        _require(1 <= C <= 32 and 1 <= G <= 32, f"pd_kl: G={G} C={C} (<= 32)")
        M = post.shape[0]
        lp, p = _group_softmax(post, G, C)
        lq, q = _group_softmax(prior, G, C)
        klg = (p * (lp - lq)).sum(-1)  # (M,G)
        kl_exact.copy_(klg.sum(-1))
        ent_post.copy_(-(p * lp).sum(-1).sum(-1))
        ent_prior.copy_(-(q * lq).sum(-1).sum(-1))
        if mode == 0:
            wpost, wprior = (1.0, 1.0) if balance < 0 else (1.0 - balance, balance)
            loss_kl.copy_(klg.sum(-1))
            dpost.copy_((wpost * p * ((lp - lq) - klg[..., None])).reshape(M, G * C))
            dprior.copy_((wprior * (q - p)).reshape(M, G * C))
        else:
            oh = F.one_hot(idx.long(), C).to(post.dtype)
            loss_kl.copy_(((lp - lq) * oh).sum(-1).sum(-1))
            dpost.copy_((oh - p).reshape(M, G * C))
            dprior.copy_((q - oh).reshape(M, G * C))

    # ------------------------------------------------------------------ conv data movement
    def im2col(self, inp, k, korder, col, round_out=True):
        NB, Hin, Win, Cc = inp.shape
        _require(Hin >= k and Win >= k, f"pd_im2col: input {Hin}x{Win}, kernel {k}")
        Ho, Wo = (Hin - k) // 2 + 1, (Win - k) // 2 + 1
        # patches[n, oy, ox, kh, kw, c]
        p = inp.unfold(1, k, 2).unfold(2, k, 2)  # (NB, Ho, Wo, C, kh, kw)
        if korder == 0:
            p = p.permute(0, 1, 2, 4, 5, 3)
        col.copy_(p.reshape(NB * Ho * Wo, k * k * Cc))

    @staticmethod
    def _col2im(col, NB, Hin, Win, Hout, Wout, Cc, k):
        c6 = col.reshape(NB, Hin, Win, k, k, Cc)
        out = torch.zeros(NB, max(Hout, (Hin - 1) * 2 + k), max(Wout, (Win - 1) * 2 + k), Cc, dtype=col.dtype,
                          device=col.device)
        for kh in range(k):
            for kw in range(k):
                out[:, kh:kh + 2 * Hin:2, kw:kw + 2 * Win:2, :] += c6[:, :, :, kh, kw, :]
        return out[:, :Hout, :Wout]

    def col2im(self, col, Hin, Win, k, bias, act, out, round_out=True):
        NB, Hout, Wout, Cc = out.shape
        sN, sY, sX, sC = out.stride()
        _require(col.dtype != torch.float16 or (sC == 1 and Cc % 4 == 0 and sN % 4 == 0 and sY % 4 == 0 and sX % 4 == 0 and
                                                _ld(col) % 4 == 0 and _aligned(out) and _aligned(col, 8) and _aligned(bias)),
                 f"pd_col2im: fp16 column matrix with Cc={Cc}, strides {out.stride()}")
        v = self._col2im(col.to(out.dtype), NB, Hin, Win, Hout, Wout, Cc, k)            # (fp16 column matrices are summed in fp32)
        if bias is not None:
            v = v + bias
        out.copy_(_act(v, act))

    def col2im_imgloss(self, col, NB, Hin, Win, Cc, k, bias, target, tgt_div, dec, diff, loss, csum):
        _require(1 <= Cc <= 16, f"pd_col2im_imgloss: {Cc} image channels (1..16)")
        Hout, Wout = (Hin - 1) * 2 + k, (Win - 1) * 2 + k
        v = self._col2im(col.to(dec.dtype), NB, Hin, Win, Hout, Wout, Cc, k) + bias  # NHWC
        v = v.permute(0, 3, 1, 2)  # NCHW
        tg = target.reshape(-1, Cc, Hout, Wout)[torch.arange(NB, device=col.device) // tgt_div]
        d = v - tg
        dec.view(NB, Cc, Hout, Wout).copy_(v)
        diff.view(NB, Cc, Hout, Wout).copy_(d)
        loss.copy_(0.5 * (d * d).sum((1, 2, 3)))
        csum.view(NB, Cc).copy_(d.sum((2, 3)))

    def bias_act_bwd(self, dy, y, act, db):
        if act == ACT_ELU:
            dy.mul_(_elu_grad_from_out(y))
        if db is not None:
            db.add_(dy.sum(0))

    def gemm_actbwd(self, A, B, C, dact, dbias, *, a_mn=False, b_mn=False):
        self.gemm(A, B, C, a_mn=a_mn, b_mn=b_mn)
        self.bias_act_bwd(C, dact, ACT_ELU, dbias)
        return C

    def conv_gemm_actbwd(self, X, k, O, Cmat, dact, dbias, *, o_mn=False):
        self.conv_gemm(1, X, k, O, Cmat, o_mn=o_mn)
        self.bias_act_bwd(Cmat, dact, ACT_ELU, dbias)
        return Cmat

    def col2im_actbwd(self, col, Hin, Win, k, dact, dbias, out):
        _require(out.shape[3] >= 1 and 1 <= k <= 6, f"pd_col2im_actbwd: Cc={out.shape[3]} k={k}")
        _require(out.shape[1] >= (Hin - 1) * 2 + k and out.shape[2] >= (Win - 1) * 2 + k,
                 "pd_col2im_actbwd: output smaller than the fold")
        self.col2im(col, Hin, Win, k, None, ACT_NONE, out, round_out=False)
        NB, Hout, Wout, Cc = out.shape
        self.bias_act_bwd(out.view(-1, Cc), dact.reshape(-1, Cc), ACT_ELU, dbias)

    def permute4(self, inp, out, perm, accumulate=False, round_out=False):
        v = inp.permute(*perm)
        if accumulate:
            out.add_(v)
        else:
            out.copy_(v)

    # ------------------------------------------------------------------ small ops
    def round_copy(self, src, dst, round_out=True):
        dst.copy_(src)

    def mask_rows(self, x, mask, out):
        out.copy_(x * mask[:, None])

    def rowscale(self, x, scale, scale_div=1, alpha=1.0):
        rows = torch.arange(x.shape[0], device=x.device) // scale_div
        x.mul_(alpha * scale[rows][:, None])

    def scale_by(self, x, scale=None, alpha=1.0):
        x.mul_(alpha * (scale.reshape(-1)[0] if scale is not None else 1.0))

    def gather_rows(self, idx, W, out):
        _require(out.shape[1] % 4 == 0 and _ld(W) % 4 == 0 and _ld(out) % 4 == 0 and _aligned(W) and _aligned(out),
                 f"pd_gather_rows: N={out.shape[1]}, ldw={_ld(W)}, ldo={_ld(out)} (% 4) / alignment")
        out.copy_(W[idx.long().reshape(-1)])

    def group_sum(self, x, I, out):
        R, W = out.shape
        out.copy_(x[:, :W].reshape(R, I, W).sum(1))

    def colsum(self, x, out):
        out.add_(x.sum(0))

    def fill(self, x, v=0.0):
        x.fill_(v)

    def reset_mask(self, reset, I, mask):
        T, B = reset.shape
        mask.view(T, B, I).copy_((~reset.bool()).to(mask.dtype)[:, :, None].expand(T, B, I))

    def scalar_head_loss(self, kind, y, target, tgt_div, loss, dy, rec):
        yy = y.reshape(-1)
        t = target.reshape(-1)[torch.arange(yy.numel(), device=y.device) // tgt_div]
        if kind == 0:
            d = t - yy
            loss.copy_(0.5 * d * d)
            dy.view(-1).copy_(-d)
            if rec is not None:
                rec.copy_(yy)
        else:
            loss.copy_(F.binary_cross_entropy_with_logits(yy, t, reduction="none"))
            s = torch.sigmoid(yy)
            dy.view(-1).copy_(s - t)
            if rec is not None:
                rec.copy_(s)

    @staticmethod
    def _nlae(v):  # -logavgexp(-v) over last dim
        I = v.shape[-1]
        if I == 1:
            return v[..., 0]
        return -((-v).logsumexp(-1) - math.log(I))

    def wm_loss(self, TB, I, kl_weight, w_img, w_rew, w_term, l_img, l_rew, l_term, l_kl, kl_exact, ent_prior,
                ent_post, w, tb):
        L = (kl_weight * l_kl + w_img * l_img + w_rew * l_rew + w_term * l_term).view(TB, I)
        tb[:, 0] = self._nlae(L)
        if I == 1:
            w.fill_(1.0 / TB)
        else:
            w.view(TB, I).copy_(F.softmax(-L, -1) / TB)
        tb[:, 1] = self._nlae(l_img.view(TB, I))
        tb[:, 2] = self._nlae(l_rew.view(TB, I))
        tb[:, 3] = self._nlae(l_term.view(TB, I))
        tb[:, 4] = self._nlae(kl_exact.view(TB, I))
        tb[:, 5] = ent_prior.view(TB, I).mean(-1)
        tb[:, 6] = ent_post.view(TB, I).mean(-1)
        tb[:, 7] = 0

    def colmean(self, x, out):
        _require(1 <= x.shape[1] <= 32, f"pd_colmean: N={x.shape[1]} (1..32)")
        out.copy_(x.mean(0))

    # ------------------------------------------------------------------ actor critic
    def gae_critic(self, H, Md, gamma, lam, vt, v, rew, term_logit, term, adv, agae, target, weight, dv, sums):
        _require(1 <= H <= 127, f"pd_gae_critic: H={H} (1..127)")
        J = H + 1
        vt, v, rew = vt.view(J, Md), v.view(J, Md), rew.view(J, Md)
        tm = torch.sigmoid(term_logit.view(J, Md))
        term.view(J, Md).copy_(tm)
        r1, t0, t1 = rew[1:], tm[:-1], tm[1:]
        a = -vt[:-1] + r1 + gamma * (1.0 - t1) * vt[1:]
        ag = torch.zeros_like(a)
        last = None
        for j in reversed(range(H)):
            last = a[j] if last is None else a[j] + lam * gamma * (1.0 - t1[j]) * last
            ag[j] = last
        tgt = ag + vt[:-1]
        wgt = (1 - t0).log().cumsum(0).exp()
        d = tgt - v[:-1]
        adv.view(H, Md).copy_(a)
        agae.view(H, Md).copy_(ag)
        target.view(H, Md).copy_(tgt)
        weight.view(H, Md).copy_(wgt)
        dv.view(H, Md).copy_(-d * wgt / (H * Md))
        s = torch.stack([(0.5 * d * d * wgt).sum(), v[0].sum(), v[:-1].sum(), r1.sum(), (r1 * r1).sum()]).double()
        sums[:5] += s

    def actor_loss_onehot(self, eta, logits, actions, agae, weight, dlogits, sums):
        rows, A = actions.shape
        _require(1 <= A <= 32, f"pd_actor_loss_onehot: A={A} (<= 32)")
        lg = logits[:, :A]
        lp = lg - lg.logsumexp(-1, keepdim=True)
        p = lp.exp()
        k = actions.argmax(-1)
        oh = F.one_hot(k, A).to(lg.dtype)
        lpa = (lp * oh).sum(-1)
        ent = -(p * lp).sum(-1)
        ag, w = agae.reshape(-1), weight.reshape(-1)
        dl = (w / rows)[:, None] * (-ag[:, None] * (oh - p) + eta * p * (lp + ent[:, None]))
        dlogits[:, :A] = dl
        sums[0] += ((-lpa * ag - eta * ent) * w).sum().double()
        sums[1] += ent.sum().double()

    def actor_loss_tanh_normal(self, eta, out, actions, agae, weight, dout, sums):
        rows, A = actions.shape
        m_, s_ = out[:, :A], out[:, A:2 * A]
        th = torch.tanh(m_ / 5)
        mu = 5 * th
        sd = F.softplus(s_) + 0.1
        eps = torch.finfo(torch.float32).eps
        y = actions.clamp(-1 + eps, 1 - eps)
        x = torch.atanh(y)
        zc = (x - mu) / sd
        lpn = -0.5 * zc * zc - sd.log() - 0.5 * math.log(2 * math.pi)
        ladj = 2.0 * (math.log(2.0) - x - F.softplus(-2.0 * x))
        lp = (lpn - ladj).sum(-1)
        ent = (0.5 + 0.5 * math.log(2 * math.pi) + sd.log()).sum(-1)
        ag, w = agae.reshape(-1), weight.reshape(-1)
        c = (w / rows)[:, None]
        dout[:, :A] = c * (-ag[:, None] * (zc / sd)) * (1 - th * th)
        dout[:, A:2 * A] = c * (-ag[:, None] * ((zc * zc - 1) / sd) - eta / sd) * torch.sigmoid(s_)
        sums[0] += ((-lp * ag - eta * ent) * w).sum().double()
        sums[1] += ent.sum().double()

    def tanh_normal_sample(self, out, eps, action):
        rows, A = action.shape
        mu = 5 * torch.tanh(out[:, :A] / 5)
        sd = F.softplus(out[:, A:2 * A]) + 0.1
        action.copy_(torch.tanh(mu + sd * eps.reshape(rows, A)))

    # ------------------------------------------------------------------ preprocessing (preprocessing.py:21-29,135-138)
    def image_u8_to_f32(self, src, dst):
        x = src.to(torch.float32) / 255.0 - 0.5
        dst.copy_(x.movedim(-1, -3))

    def onehot_i64(self, idx, out):
        out.copy_(F.one_hot(idx.long(), out.shape[-1]).to(out.dtype))

    def tanh(self, x, y):
        y.copy_(torch.tanh(x))

    # ------------------------------------------------------------------ optimizer
    def sumsq(self, x, out):
        out.add_((x * x).sum())

    def clip_scale(self, x, sumsq, max_norm, norm_out):
        norm = sumsq.sqrt()
        coef = torch.clamp(max_norm / (norm + 1e-6), max=1.0)
        x.mul_(coef)
        if norm_out is not None:
            norm_out.copy_(norm.reshape(norm_out.shape))

    def adamw(self, p, g, m, v, lr, beta1, beta2, eps, wd, step):
        st = float(step.item())
        p.mul_(1 - lr * wd)
        m.lerp_(g, 1 - beta1)
        v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
        bc1 = 1 - beta1 ** st
        bc2s = math.sqrt(1 - beta2 ** st)
        p.addcdiv_(m, v.sqrt() / bc2s + eps, value=-lr / bc1)

    def inc(self, counter):
        counter.add_(1)
