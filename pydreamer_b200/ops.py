"""Tensor-level wrappers over the C ABI (include/pd_b200.h).

`NativeOps` is the product path: every method enqueues one hand-written sm_90a kernel on the
current CUDA stream through libpd_b200.so.  There is no CPU implementation in this package: the
constructor raises if CUDA or the library is unavailable.

Tests may install a reference implementation of the *same interface* (oracle/ref_ops.py, plain
torch) with `set_ops_for_testing` to check the host-side composition and hand-written backward of
pydreamer_b200.dreamer on CPU; that hook is refused unless PD_B200_TESTING=1 is set by the test
harness, so a product run can never route through it.
"""
import ctypes
import os

import torch

from . import _native

ACT_NONE, ACT_ELU = 0, 1
GEMM_TC, GEMM_SIMT = 0, 1
SUPPORT_MAX = 1024                      # PD_SUPPORT_MAX: the widest categorical reward support pd_support_head takes


_cur_dev = getattr(torch._C, "_cuda_getDevice", None) or torch.cuda.current_device    # the raw binding: no lazy-init checks per launch


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _ld(t):
    """Row stride (elements) of a 2-D view whose last dim is contiguous."""
    assert t.dim() == 2 and (t.shape[1] == 1 or t.stride(1) == 1), (t.shape, t.stride())
    return t.stride(0) if t.shape[0] > 1 else max(t.stride(0), t.shape[1])


class RssmFwdArgs(ctypes.Structure):
    """struct pd_rssm_fwd_args of include/pd_b200.h (same field order)."""
    _INTS = ("T", "BI", "I", "D", "Hd", "G", "C")
    _PTRS1 = ("w_z16", "w_ih16", "w_hh16", "w_ph16", "w_pm16", "b_z", "ln1_g", "ln1_b", "b_ih", "b_hh", "b_ph",
              "ln2_g", "ln2_b", "b_pm")
    _PTRS2 = ("aa", "ea", "mask", "noise", "x1", "za", "m1", "r1", "gates", "feat", "hin", "zin", "y2", "pin", "m2",
              "r2", "post", "idx", "ws_wzT16", "ws_za16", "ws_h16", "ws_pin16", "ws_barrier", "ws_ghpart", "ws_y2part")
    _LAYERS = ("w_ih16_l", "b_ih_l", "b_hh_l")                 # stacked GRU: layers 1 .. L-1
    _fields_ = ([(n, ctypes.c_int) for n in _INTS] + [(n, ctypes.c_void_p) for n in _PTRS1] +
                [("eps", ctypes.c_float)] + [(n, ctypes.c_void_p) for n in _PTRS2] + [("layers", ctypes.c_int)] +
                [(n, ctypes.c_void_p * 3) for n in _LAYERS])


class RssmBwdArgs(ctypes.Structure):
    """struct pd_rssm_bwd_args of include/pd_b200.h (same field order)."""
    _INTS = ("T", "BI", "D", "Hd", "G", "C", "round_out", "ks2", "ks6")
    _PTRS = ("w_pmT16", "w_phT16", "w_hhT16", "w_ihT16", "w_zT16", "ln2_g", "ln1_g", "post", "pin", "y2", "m2", "r2", "x1", "za",
             "m1", "r1", "gates", "hin", "mask", "dfeat", "dpost_u", "w", "dpost", "dy2", "dgi", "dgh", "dx1", "g_ln2_g",
             "g_ln2_b", "g_b_ph", "g_ln1_g", "g_ln1_b", "g_b_z", "ws_part2", "ws_part6", "ws_part7", "ws_barrier")
    _fields_ = ([(n, ctypes.c_int) for n in _INTS] + [("kl_weight", ctypes.c_float)] + [(n, ctypes.c_void_p) for n in _PTRS])


class NativeOps:
    """One library handle on one device.  Its fixed-order gradient reductions use a 16 MB scratch area per stream, for up
    to eight streams (128 MB of device memory, allocated here); a reduction on a ninth stream raises."""
    is_reference = False

    def __init__(self, device):
        device = torch.device(device)
        if device.type != "cuda" or not torch.cuda.is_available():
            raise RuntimeError("pydreamer_b200 needs a CUDA (sm_90a) device: there is no CPU fallback")
        self.device = device
        self.lib = _native.load()
        h = ctypes.c_void_p()
        idx = device.index if device.index is not None else torch.cuda.current_device()
        rc = self.lib.pd_create(int(idx), ctypes.byref(h))
        if rc != 0:
            raise RuntimeError(f"pd_create failed ({rc}): device {idx} is not an sm_90 (H100) GPU or the driver is too old")
        self.h = h
        self._index = int(idx)
        self.gemm_profile = None   # list of (start_event, end_event, flops, shape key) when bench.py profiles a step

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.pd_destroy(self.h)
        except Exception:
            pass

    # ------------------------------------------------------------------ plumbing
    def _s(self):
        # kernels launch on the CURRENT device: refuse to enqueue this handle's work on another GPU's context
        if _cur_dev() != self._index:
            raise RuntimeError(f"pydreamer_b200: current CUDA device is {torch.cuda.current_device()} but this model lives on "
                               f"cuda:{self._index}; wrap the call in `with torch.cuda.device({self._index})`")
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _ck(self, rc, name):
        if rc != 0:
            raise RuntimeError(f"{name} failed ({rc}): {self.lib.pd_last_error(self.h).decode()}")

    def set_gemm_impl(self, impl):
        self._ck(self.lib.pd_set_gemm_impl(self.h, int(impl)), "pd_set_gemm_impl")

    def set_round_operands(self, on):
        self._ck(self.lib.pd_set_round_operands(self.h, int(bool(on))), "pd_set_round_operands")

    def launch_count(self):
        return int(self.lib.pd_launch_count(self.h))

    def _profiled(self, launch, flops, shape):
        """Runs launch().  While bench.py profiles a step (gemm_profile is a list), the launch is bracketed by CUDA events
        and (start_event, end_event, flops, shape key) is appended to gemm_profile."""
        prof = self.gemm_profile
        if prof is None:
            return launch()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        launch()
        e1.record()
        prof.append((e0, e1, flops, shape))

    # ------------------------------------------------------------------ gemm
    def gemm(self, A, B, C, *, a_mn=False, b_mn=False, bias=None, res=None, r_div=1, act=ACT_NONE,
             round_out=False, accumulate=False, c_zeroed=False):
        """C[M,N] (=|+=) A(m,k) B(n,k).  A: [M,K] (or stored [K,M] if a_mn); B: [N,K] (or [K,N] if b_mn)."""
        M, N = C.shape
        K = A.shape[0] if a_mn else A.shape[1]
        assert (A.shape[1] if a_mn else A.shape[0]) == M, (A.shape, C.shape, a_mn)
        assert (B.shape == (K, N)) if b_mn else (B.shape == (N, K)), (B.shape, (N, K), b_mn)
        flags = (1 if c_zeroed else 0) | (2 if C.dtype == torch.float16 else 0)       # PD_GEMM_C_ZEROED | PD_GEMM_C_F16
        self._profiled(lambda: self._ck(self.lib.pd_gemm(
            self.h, M, N, K, _ptr(A), _ld(A), int(a_mn), _ptr(B), _ld(B), int(b_mn), _ptr(C), _ld(C), _ptr(bias), _ptr(res),
            _ld(res) if res is not None else 0, int(r_div), int(act), int(round_out), int(accumulate), flags, self._s()),
            "pd_gemm"), 2.0 * M * N * K, (M, N, K, int(a_mn), int(b_mn), int(accumulate)))
        return C

    def gemm_f16(self, A16, B16, C, *, bias=None, res=None, r_div=1, act=ACT_NONE, round_out=False):
        """C[M,N] (fp32) = A16[M,K] B16[N,K]^T with fp16 operands (forward-only layers)."""
        M, N = C.shape
        K = A16.shape[1]
        assert A16.dtype == torch.float16 and B16.dtype == torch.float16 and B16.shape == (N, K) and A16.shape[0] == M
        self._profiled(lambda: self._ck(self.lib.pd_gemm_f16(
            self.h, M, N, K, _ptr(A16), _ld(A16), _ptr(B16), _ld(B16), _ptr(C), _ld(C), _ptr(bias), _ptr(res),
            _ld(res) if res is not None else 0, int(r_div), int(act), int(round_out), self._s()), "pd_gemm_f16"),
            2.0 * M * N * K, (M, N, K, "f16", 0, 0))
        return C

    def conv_gemm(self, mode, X, k, O, Cmat, *, o_mn=False, bias=None, act=ACT_NONE, round_out=False):
        """Implicit-GEMM convolution contraction (pd_conv_gemm): X is a contiguous NHWC tensor (NB,H,W,C)."""
        NB, H, W, C = X.shape
        assert X.is_contiguous()
        odim = Cmat.shape[1] if mode in (1, 2) else Cmat.shape[0]
        P, Q = (H - k) // 2 + 1, (W - k) // 2 + 1
        self._profiled(lambda: self._ck(self.lib.pd_conv_gemm(
            self.h, int(mode), NB, H, W, C, int(k), _ptr(X), _ptr(O), _ld(O), int(o_mn), odim, _ptr(Cmat), _ld(Cmat),
            _ptr(bias), int(act), int(round_out), 0 if mode == 1 else 1, self._s()), "pd_conv_gemm"),
            2.0 * NB * P * Q * k * k * C * odim, (NB * P * Q, odim, k * k * C, f"conv{mode}", int(o_mn), 0))
        return Cmat

    def to_half(self, src, dst):
        M, N = src.shape
        self._ck(self.lib.pd_to_half(self.h, M, N, _ptr(src), _ld(src), _ptr(dst), _ld(dst), self._s()), "pd_to_half")

    # ------------------------------------------------------------------ rowwise
    def ln_elu_fwd(self, x, gamma, beta, eps, y, mean, rstd, y16=None):
        M, N = x.shape
        self._ck(self.lib.pd_ln_elu_fwd(self.h, M, N, _ptr(x), _ld(x), _ptr(gamma), _ptr(beta), float(eps),
                                        _ptr(y), _ld(y), _ptr(mean), _ptr(rstd), _ptr(y16),
                                        _ld(y16) if y16 is not None else 0, self._s()), "pd_ln_elu_fwd")

    def ln_elu_bwd(self, dy, x, y, gamma, mean, rstd, dx, dgamma, dbeta, dbias=None):
        M, N = x.shape
        self._ck(self.lib.pd_ln_elu_bwd(self.h, M, N, _ptr(dy), _ld(dy), _ptr(x), _ld(x), _ptr(y), _ld(y),
                                        _ptr(gamma), _ptr(mean), _ptr(rstd), _ptr(dx), _ld(dx), _ptr(dgamma),
                                        _ptr(dbeta), _ptr(dbias), self._s()), "pd_ln_elu_bwd")

    def gru_fwd(self, gi, gh, hprev, hout, hmask=None, mask_next=None, gates=None, h16=None):
        M, D = hprev.shape
        self._ck(self.lib.pd_gru_fwd(self.h, M, D, _ptr(gi), _ld(gi), _ptr(gh), _ld(gh), _ptr(hprev), _ld(hprev),
                                     _ptr(hout), _ld(hout), _ptr(hmask), _ld(hmask) if hmask is not None else 0,
                                     _ptr(mask_next), _ptr(gates), _ptr(h16), _ld(h16) if h16 is not None else 0,
                                     self._s()), "pd_gru_fwd")

    def gru_bwd(self, dh_a, dh_b, mask_b, gates, hprev, dgi, dgh, dh_carry):
        M, D = hprev.shape
        self._ck(self.lib.pd_gru_bwd(self.h, M, D, _ptr(dh_a), _ld(dh_a) if dh_a is not None else 0, _ptr(dh_b),
                                     _ld(dh_b) if dh_b is not None else 0, _ptr(mask_b), _ptr(gates), _ptr(hprev),
                                     _ld(hprev), _ptr(dgi), _ld(dgi), _ptr(dgh), _ld(dgh), _ptr(dh_carry),
                                     _ld(dh_carry), self._s()), "pd_gru_bwd")

    def rssm_unroll_fwd(self, dims, eps, **t):
        """Persistent posterior unroll (pd_rssm_unroll_fwd).  dims = dict(T, BI, I, D, Hd, G, C, optional layers); every
        other struct field is passed as a contiguous tensor (or None) by its field name, the per-layer ones (w_ih16_l,
        b_ih_l, b_hh_l) as lists of the tensors of layers 1 .. L-1."""
        a = RssmFwdArgs()
        for n in RssmFwdArgs._INTS:
            setattr(a, n, int(dims[n]))
        a.eps = float(eps)
        a.layers = int(dims.get("layers", 0))
        for n in RssmFwdArgs._LAYERS:
            for i, v in enumerate(t.pop(n, None) or ()):
                assert v.is_contiguous(), n
                getattr(a, n)[i] = v.data_ptr()
        for n in RssmFwdArgs._PTRS1 + RssmFwdArgs._PTRS2:
            v = t.pop(n, None)
            if v is not None:
                assert v.is_contiguous(), n
                setattr(a, n, v.data_ptr())
        assert not t, f"unknown fields {sorted(t)}"
        self._ck(self.lib.pd_rssm_unroll_fwd(self.h, ctypes.byref(a), self._s()), "pd_rssm_unroll_fwd")

    def rssm_unroll_bwd(self, dims, kl_weight, round_out=True, **t):
        """Persistent BPTT of the posterior unroll (pd_rssm_unroll_bwd).  dims = dict(T, BI, D, Hd, G, C); every pointer
        field of the struct is passed as a contiguous tensor by its field name."""
        a = RssmBwdArgs()
        for n in ("T", "BI", "D", "Hd", "G", "C"):
            setattr(a, n, int(dims[n]))
        a.round_out = int(bool(round_out))
        a.kl_weight = float(kl_weight)
        for n in RssmBwdArgs._PTRS:
            v = t.pop(n)
            assert v.is_contiguous(), n
            setattr(a, n, v.data_ptr())
        assert not t, f"unknown fields {sorted(t)}"
        self._ck(self.lib.pd_rssm_unroll_bwd(self.h, ctypes.byref(a), self._s()), "pd_rssm_unroll_bwd")

    def transpose_to_half(self, src, dst):
        """dst[n, m] (fp16) = src[m, n] (fp32)"""
        M, N = src.shape
        assert dst.shape == (N, M) and dst.dtype == torch.float16
        self._ck(self.lib.pd_transpose_to_half(self.h, M, N, _ptr(src), _ld(src), _ptr(dst), _ld(dst), self._s()),
                 "pd_transpose_to_half")

    def cat_sample(self, logits, noise, G, C, z, zmask=None, mask_next=None, idx=None, z16=None):
        M = logits.shape[0]
        self._ck(self.lib.pd_cat_sample(self.h, M, G, C, _ptr(logits), _ld(logits), _ptr(noise), _ld(noise), _ptr(z),
                                        _ld(z), _ptr(zmask), _ld(zmask) if zmask is not None else 0, _ptr(mask_next),
                                        _ptr(idx), _ptr(z16), _ld(z16) if z16 is not None else 0, self._s()),
                 "pd_cat_sample")

    def cat_st_bwd(self, logits, G, C, dz_a, dz_b, mask_b, extra, rowscale, alpha, dlogits):
        M = logits.shape[0]
        self._ck(self.lib.pd_cat_st_bwd(self.h, M, G, C, _ptr(logits), _ld(logits), _ptr(dz_a),
                                        _ld(dz_a) if dz_a is not None else 0, _ptr(dz_b),
                                        _ld(dz_b) if dz_b is not None else 0, _ptr(mask_b), _ptr(extra),
                                        _ld(extra) if extra is not None else 0, _ptr(rowscale), float(alpha),
                                        _ptr(dlogits), _ld(dlogits), self._s()), "pd_cat_st_bwd")

    def kl(self, post, prior, idx, mode, balance, G, C, loss_kl, kl_exact, ent_post, ent_prior, dpost, dprior):
        M = post.shape[0]
        self._ck(self.lib.pd_kl(self.h, M, G, C, _ptr(post), _ld(post), _ptr(prior), _ld(prior), _ptr(idx), int(mode),
                                float(balance), _ptr(loss_kl), _ptr(kl_exact), _ptr(ent_post), _ptr(ent_prior),
                                _ptr(dpost), _ld(dpost), _ptr(dprior), _ld(dprior), self._s()), "pd_kl")

    # ------------------------------------------------------------------ conv data movement
    def im2col(self, inp, k, korder, col, round_out=True):
        """inp: 4-D view indexed [n, y, x, c] (any strides); col: [NB*Ho*Wo, k*k*C]."""
        NB, Hin, Win, Cc = inp.shape
        sN, sY, sX, sC = inp.stride()
        self._ck(self.lib.pd_im2col(self.h, NB, Hin, Win, Cc, k, korder, _ptr(inp), sN, sY, sX, sC, _ptr(col),
                                    _ld(col), int(round_out), self._s()), "pd_im2col")

    def col2im(self, col, Hin, Win, k, bias, act, out, round_out=True):
        """out: 4-D view indexed [n, y, x, c]; col: [NB*Hin*Win, k*k*C]."""
        NB, Hout, Wout, Cc = out.shape
        sN, sY, sX, sC = out.stride()
        self._ck(self.lib.pd_col2im_t(self.h, NB, Hin, Win, Hout, Wout, Cc, k, _ptr(col), _ld(col),
                                      int(col.dtype == torch.float16), _ptr(bias), int(act), int(round_out), _ptr(out), sN, sY,
                                      sX, sC, self._s()), "pd_col2im")

    def col2im_imgloss(self, col, NB, Hin, Win, Cc, k, bias, target, tgt_div, dec, diff, loss, csum):
        self._ck(self.lib.pd_col2im_imgloss_t(self.h, NB, Hin, Win, Cc, k, _ptr(col), _ld(col),
                                              int(col.dtype == torch.float16), _ptr(bias), _ptr(target), int(tgt_div),
                                              _ptr(dec), _ptr(diff), _ptr(loss), _ptr(csum), self._s()), "pd_col2im_imgloss")

    def bias_act_bwd(self, dy, y, act, db):
        M, N = dy.shape
        self._ck(self.lib.pd_bias_act_bwd(self.h, M, N, _ptr(dy), _ld(dy), _ptr(y), _ld(y) if y is not None else 0,
                                          int(act), _ptr(db), self._s()), "pd_bias_act_bwd")

    def gemm_actbwd(self, A, B, C, dact, dbias, *, a_mn=False, b_mn=False):
        """C = (A B^T) * elu'(dact); dbias += column sums (pd_gemm_actbwd: GEMM + bias_act_bwd in one launch)."""
        M, N = C.shape
        K = A.shape[0] if a_mn else A.shape[1]
        self._profiled(lambda: self._ck(self.lib.pd_gemm_actbwd(
            self.h, M, N, K, _ptr(A), _ld(A), int(a_mn), _ptr(B), _ld(B), int(b_mn), _ptr(C), _ld(C), _ptr(dact), _ld(dact),
            _ptr(dbias), self._s()), "pd_gemm_actbwd"), 2.0 * M * N * K, (M, N, K, int(a_mn), int(b_mn), 0))
        return C

    def conv_gemm_actbwd(self, X, k, O, Cmat, dact, dbias, *, o_mn=False):
        """pd_conv_gemm mode 1 followed by the ELU backward of the layer below and its bias gradient, one launch."""
        NB, H, W, C = X.shape
        assert X.is_contiguous()
        odim = Cmat.shape[1]
        P, Q = (H - k) // 2 + 1, (W - k) // 2 + 1
        self._profiled(lambda: self._ck(self.lib.pd_conv_gemm_actbwd(
            self.h, NB, H, W, C, int(k), _ptr(X), _ptr(O), _ld(O), int(o_mn), odim, _ptr(Cmat), _ld(Cmat), _ptr(dact),
            _ld(dact), _ptr(dbias), self._s()), "pd_conv_gemm_actbwd"),
            2.0 * NB * P * Q * k * k * C * odim, (NB * P * Q, odim, k * k * C, "conv1", int(o_mn), 0))
        return Cmat

    def col2im_actbwd(self, col, Hin, Win, k, dact, dbias, out):
        """out (NB,Hout,Wout,Cc contiguous) = fold(col) * elu'(dact); dbias += per-channel sums (pd_col2im_actbwd)."""
        NB, Hout, Wout, Cc = out.shape
        assert out.is_contiguous() and dact.is_contiguous() and dact.numel() == out.numel()
        self._ck(self.lib.pd_col2im_actbwd(self.h, NB, Hin, Win, Hout, Wout, Cc, int(k), _ptr(col), _ld(col), _ptr(dact), _ptr(dbias),
                                           _ptr(out), self._s()), "pd_col2im_actbwd")

    def permute4(self, inp, out, perm, accumulate=False, round_out=False):
        """out (contiguous, shape = inp.shape permuted by perm) (+)= inp.permute(perm)."""
        assert out.is_contiguous() and inp.dim() == 4
        dims = (ctypes.c_int * 4)(*inp.shape)
        pm = (ctypes.c_int * 4)(*perm)
        st = None if inp.is_contiguous() else (ctypes.c_long * 4)(*inp.stride())
        self._ck(self.lib.pd_permute4(self.h, _ptr(inp), _ptr(out), dims, pm, st, int(accumulate), int(round_out),
                                      self._s()), "pd_permute4")

    # ------------------------------------------------------------------ small ops
    def round_copy(self, src, dst, round_out=True):
        assert src.is_contiguous() and dst.is_contiguous()
        self._ck(self.lib.pd_round_copy(self.h, _ptr(src), _ptr(dst), src.numel(), int(round_out), self._s()),
                 "pd_round_copy")

    def mask_rows(self, x, mask, out):
        M, N = x.shape
        self._ck(self.lib.pd_mask_rows(self.h, M, N, _ptr(x), _ld(x), _ptr(mask), _ptr(out), _ld(out), self._s()),
                 "pd_mask_rows")

    def rowscale(self, x, scale, scale_div=1, alpha=1.0):
        M, N = x.shape
        self._ck(self.lib.pd_rowscale(self.h, M, N, _ptr(x), _ld(x), _ptr(scale), int(scale_div), float(alpha),
                                      self._s()), "pd_rowscale")

    def scale_by(self, x, scale=None, alpha=1.0):
        """x *= alpha * scale[0] (no operand rounding; a factor of exactly 1 is a no-op on the device)."""
        assert x.is_contiguous()
        self._ck(self.lib.pd_scale_by(self.h, _ptr(x), x.numel(), _ptr(scale), float(alpha), self._s()), "pd_scale_by")

    def gather_rows(self, idx, W, out):
        """out[m, :] = W[idx[m], :]  (idx int32 [M], W [rows, N], out [M, N])"""
        M, N = out.shape
        assert idx.dtype == torch.int32 and idx.is_contiguous() and idx.numel() == M
        self._ck(self.lib.pd_gather_rows(self.h, M, N, _ptr(idx), _ptr(W), _ld(W), _ptr(out), _ld(out), self._s()),
                 "pd_gather_rows")

    def group_sum(self, x, I, out):
        R, W = out.shape
        self._ck(self.lib.pd_group_sum(self.h, R, I, W, _ptr(x), _ld(x), _ptr(out), _ld(out), self._s()),
                 "pd_group_sum")

    def colsum(self, x, out):
        M, N = x.shape
        self._ck(self.lib.pd_colsum(self.h, M, N, _ptr(x), _ld(x), _ptr(out), self._s()), "pd_colsum")

    def fill(self, x, v=0.0):
        assert x.is_contiguous()
        self._ck(self.lib.pd_fill(self.h, _ptr(x), x.numel(), float(v), self._s()), "pd_fill")

    def reset_mask(self, reset, I, mask):
        T, B = reset.shape
        r = reset.contiguous().view(torch.uint8) if reset.dtype == torch.bool else reset.to(torch.uint8)
        self._ck(self.lib.pd_reset_mask(self.h, T, B, I, _ptr(r), _ptr(mask), self._s()), "pd_reset_mask")

    def scalar_head_loss(self, kind, y, target, tgt_div, loss, dy, rec):
        self._ck(self.lib.pd_scalar_head_loss(self.h, y.numel(), int(kind), _ptr(y), _ptr(target), int(tgt_div),
                                              _ptr(loss), _ptr(dy), _ptr(rec), self._s()), "pd_scalar_head_loss")

    def vec_head_loss(self, y, target, tgt_div, loss, dy):
        """loss[m] = 0.5 sum_k (target[m / tgt_div, k] - y[m, k])^2, dy = y - target (row-strided 2-D views)."""
        M, K = y.shape
        assert target.shape[1] == K and dy.shape == (M, K) and loss.numel() == M
        self._ck(self.lib.pd_vec_head_loss(self.h, M, K, _ptr(y), _ld(y), _ptr(target), _ld(target), int(tgt_div),
                                           _ptr(loss), _ptr(dy), _ld(dy), self._s()), "pd_vec_head_loss")

    def support_head(self, y, support, target, tgt_div, rec, loss=None, dy=None, idx=None):
        """Categorical reward head (pd_support_head): rec[m] = softmax(y[m]) . support; with a target (row m reads
        target[m / tgt_div]) also loss = logsumexp(y) - y[k*], dy = softmax(y) - onehot(k*) and idx = k* (int32)."""
        M, S = y.shape
        assert support.numel() == S and (rec is None or rec.numel() == M)
        assert idx is None or (idx.dtype == torch.int32 and idx.is_contiguous() and idx.numel() == M)
        self._ck(self.lib.pd_support_head(self.h, M, S, _ptr(y), _ld(y), _ptr(support), _ptr(target), int(tgt_div),
                                          _ptr(rec), _ptr(loss), _ptr(dy), _ld(dy) if dy is not None else 0, _ptr(idx),
                                          self._s()), "pd_support_head")

    def wm_loss(self, TB, I, kl_weight, w_img, w_rew, w_term, l_img, l_rew, l_term, l_kl, kl_exact, ent_prior,
                ent_post, w, tb, l_vec=None, w_vec=0.0):
        self._ck(self.lib.pd_wm_loss(self.h, TB, I, float(kl_weight), float(w_img), float(w_rew), float(w_term),
                                     _ptr(l_img), _ptr(l_rew), _ptr(l_term), _ptr(l_kl), _ptr(kl_exact),
                                     _ptr(ent_prior), _ptr(ent_post), _ptr(l_vec), float(w_vec), _ptr(w), _ptr(tb),
                                     self._s()), "pd_wm_loss")

    def colmean(self, x, out):
        M, N = x.shape
        assert x.is_contiguous()
        self._ck(self.lib.pd_colmean(self.h, M, N, _ptr(x), _ptr(out), self._s()), "pd_colmean")

    # ------------------------------------------------------------------ actor critic
    def gae_critic(self, H, Md, gamma, lam, vt, v, rew, term_logit, term, adv, agae, target, weight, dv, sums):
        self._ck(self.lib.pd_gae_critic(self.h, H, Md, float(gamma), float(lam), _ptr(vt), _ptr(v), _ptr(rew),
                                        _ptr(term_logit), _ptr(term), _ptr(adv), _ptr(agae), _ptr(target),
                                        _ptr(weight), _ptr(dv), _ptr(sums), self._s()), "pd_gae_critic")

    def gae_critic_obs(self, T, B, gamma, lam, vt, v, rew, term, scale, dv, sums):
        """The GAE / critic-loss scan over observed rewards and 0/1 terminals (pd_gae_critic_obs): T rows of B columns;
        dv = scale * d loss_critic / d v[:-1]; sums[0:2] (float64) += {loss_critic * (T-1) B, sum v[:-1]}."""
        assert sums.dtype == torch.float64 and all(t.is_contiguous() for t in (vt, v, rew, term, dv))
        self._ck(self.lib.pd_gae_critic_obs(self.h, int(T), int(B), float(gamma), float(lam), _ptr(vt), _ptr(v), _ptr(rew),
                                            _ptr(term), float(scale), _ptr(dv), _ptr(sums), self._s()), "pd_gae_critic_obs")

    def actor_loss_onehot(self, eta, logits, actions, agae, weight, dlogits, sums):
        rows, A = actions.shape
        self._ck(self.lib.pd_actor_loss_onehot(self.h, rows, A, float(eta), _ptr(logits), _ld(logits), _ptr(actions),
                                               _ld(actions), _ptr(agae), _ptr(weight), _ptr(dlogits), _ld(dlogits),
                                               _ptr(sums), self._s()), "pd_actor_loss_onehot")

    def actor_loss_tanh_normal(self, eta, out, actions, agae, weight, dout, sums):
        rows, A = actions.shape
        self._ck(self.lib.pd_actor_loss_tanh_normal(self.h, rows, A, float(eta), _ptr(out), _ld(out), _ptr(actions),
                                                    _ld(actions), _ptr(agae), _ptr(weight), _ptr(dout), _ld(dout),
                                                    _ptr(sums), self._s()), "pd_actor_loss_tanh_normal")

    def tanh_normal_sample(self, out, eps, action):
        rows, A = action.shape
        self._ck(self.lib.pd_tanh_normal_sample(self.h, rows, A, _ptr(out), _ld(out), _ptr(eps), _ptr(action),
                                                _ld(action), self._s()), "pd_tanh_normal_sample")

    def actor_loss_normal_tanh(self, eta, out, actions, agae, weight, dout, sums):
        rows, A = actions.shape
        self._ck(self.lib.pd_actor_loss_normal_tanh(self.h, rows, A, float(eta), _ptr(out), _ld(out), _ptr(actions),
                                                    _ld(actions), _ptr(agae), _ptr(weight), _ptr(dout), _ld(dout),
                                                    _ptr(sums), self._s()), "pd_actor_loss_normal_tanh")

    def normal_tanh_sample(self, out, eps, action):
        rows, A = action.shape
        self._ck(self.lib.pd_normal_tanh_sample(self.h, rows, A, _ptr(out), _ld(out), _ptr(eps), _ptr(action),
                                                _ld(action), self._s()), "pd_normal_tanh_sample")

    # ------------------------------------------------------------------ preprocessing
    def image_u8_to_f32(self, src, dst):
        NB = src.numel() // (src.shape[-1] * src.shape[-2] * src.shape[-3])
        H, W, C = src.shape[-3:]
        self._ck(self.lib.pd_image_u8_to_f32(self.h, NB, H, W, C, _ptr(src), _ptr(dst), self._s()), "pd_image_u8_to_f32")

    def onehot_i64(self, idx, out):
        self._ck(self.lib.pd_onehot_i64(self.h, idx.numel(), out.shape[-1], _ptr(idx), _ptr(out), self._s()), "pd_onehot_i64")

    def tanh(self, x, y):
        self._ck(self.lib.pd_tanh(self.h, x.numel(), _ptr(x), _ptr(y), self._s()), "pd_tanh")

    def image_ids_onehot(self, ids, out):
        """Category ids (..., H, W) of uint8 / int32 / int64 -> fp32 one-hot out (..., C, H, W); NaN where an id is
        outside [0, C) (pd_image_ids_onehot)."""
        C, H, W = out.shape[-3:]
        assert ids.shape[-2:] == (H, W) and ids.is_contiguous() and out.is_contiguous()
        nbytes = {torch.uint8: 1, torch.int32: 4, torch.int64: 8}.get(ids.dtype)
        if nbytes is None:
            raise TypeError(f"pd_image_ids_onehot: category ids of dtype {ids.dtype} (uint8, int32 or int64)")
        self._ck(self.lib.pd_image_ids_onehot(self.h, ids.numel() // (H * W), C, H * W, _ptr(ids), nbytes, _ptr(out),
                                              self._s()), "pd_image_ids_onehot")

    # ------------------------------------------------------------------ categorical grid images
    def grid_enc_input(self, image, reward, terminal, out):
        """out[n] = [image[n] | reward[n] plane | terminal[n] plane] (pd_grid_enc_input); image (NB, C, H, W) contiguous."""
        NB, C, H, W = image.shape
        assert image.is_contiguous() and reward.is_contiguous() and terminal.is_contiguous()
        assert reward.numel() == NB and terminal.numel() == NB and out.shape == (NB, (C + 2) * H * W)
        self._ck(self.lib.pd_grid_enc_input(self.h, NB, C, H * W, _ptr(image), _ptr(reward), _ptr(terminal), _ptr(out),
                                            _ld(out), self._s()), "pd_grid_enc_input")

    def cat_image_loss(self, y, C, target, tgt_div, min_prob, loss=None, dy=None, rec=None):
        """Categorical image loss (pd_cat_image_loss): y (M, C*P) logits, target (M / tgt_div, C*P) one-hot images;
        loss (M,), dy (M, C*P) and rec (M / tgt_div, C*P) are each optional."""
        M, CP = y.shape
        assert CP % C == 0 and target.shape[1] == CP
        assert dy is None or dy.shape == (M, CP)
        assert rec is None or (rec.is_contiguous() and rec.numel() == (M // max(tgt_div, 1)) * CP)
        assert loss is None or (loss.is_contiguous() and loss.numel() == M)
        self._ck(self.lib.pd_cat_image_loss(self.h, M, C, CP // C, _ptr(y), _ld(y), _ptr(target), _ld(target), int(tgt_div),
                                            float(min_prob), _ptr(loss), _ptr(dy), _ld(dy) if dy is not None else 0,
                                            _ptr(rec), self._s()), "pd_cat_image_loss")

    # ------------------------------------------------------------------ optimizer
    def sumsq(self, x, out):
        assert x.is_contiguous()
        ws = getattr(self, "_sumsq_ws", None)
        if ws is None:
            ws = self._sumsq_ws = torch.empty(int(self.lib.pd_sumsq_ws_floats(self.h)), dtype=torch.float32, device=self.device)
        self._ck(self.lib.pd_sumsq(self.h, _ptr(x), x.numel(), _ptr(out), _ptr(ws), self._s()), "pd_sumsq")

    def clip_scale(self, x, sumsq, max_norm, norm_out):
        self._ck(self.lib.pd_clip_scale(self.h, _ptr(x), x.numel(), _ptr(sumsq), float(max_norm), _ptr(norm_out),
                                        self._s()), "pd_clip_scale")

    def adamw(self, p, g, m, v, lr, beta1, beta2, eps, wd, step):
        self._ck(self.lib.pd_adamw(self.h, _ptr(p), _ptr(g), _ptr(m), _ptr(v), p.numel(), float(lr), float(beta1),
                                   float(beta2), float(eps), float(wd), _ptr(step), self._s()), "pd_adamw")

    def inc(self, counter):
        self._ck(self.lib.pd_inc(self.h, _ptr(counter), self._s()), "pd_inc")


# ---------------------------------------------------------------------- ops registry
_TEST_OPS = None


def set_ops_for_testing(ops):
    """Install a reference op table (tests only; see module docstring)."""
    global _TEST_OPS
    if ops is not None and os.environ.get("PD_B200_TESTING") != "1":
        raise RuntimeError("set_ops_for_testing is only available to the test harness (PD_B200_TESTING=1)")
    _TEST_OPS = ops


def get_ops(device):
    if _TEST_OPS is not None:
        return _TEST_OPS
    return NativeOps(device)
