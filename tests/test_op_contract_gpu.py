"""The reference op table refuses what the native table refuses.

oracle/ref_ops.py restates the host-side argument checks (PD_REQUIRE) of each native entry point the model reaches, so
that a schedule which runs on the reference table on a CPU also passes the native checks.  Each restated condition is
called here once just inside and once just outside its boundary, on the same device tensors through both tables: they
must agree on accept or refuse, and a native refusal launches nothing."""
import pytest
import torch

from oracle.vecobs_ops import VecRefOps
from tests.test_gemm_conv_f64_gpu import refused

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
f16 = torch.float16


def z(*shape, dtype=torch.float32):
    return torch.zeros(*shape, device=DEV, dtype=dtype)


def one(*shape):
    return torch.ones(*shape, device=DEV)


def f16_gemm(M=64, N=64, K=64, lda=64, ldb=64, a_off=0):
    return lambda o: o.gemm_f16(z(M, lda + a_off, dtype=f16)[:, a_off:a_off + K], z(N, ldb, dtype=f16)[:, :K], z(M, N))


def conv(C=4, ldo=None):
    ldo = ldo or 16 * C
    return lambda o: o.conv_gemm(1, z(2, 14, 14, C), 4, z(32, ldo)[:, :16 * C], z(72, 32))


def ln_fwd(N):
    return lambda o: o.ln_elu_fwd(z(4, N), one(N), z(N), 1e-3, z(4, N), z(4), one(4))


def ln_bwd(N):
    return lambda o: o.ln_elu_bwd(z(4, N), z(4, N), z(4, N), one(N), z(4), one(4), z(4, N), z(N), z(N))


def kl(G, C):
    M = 4
    return lambda o: o.kl(z(M, G * C), z(M, G * C), None, 0, -1.0, G, C, z(M), z(M), z(M), z(M), z(M, G * C), z(M, G * C))


def imgloss(Cc):
    return lambda o: o.col2im_imgloss(z(900, 36 * Cc), 1, 30, 30, Cc, 6, z(Cc), z(1, Cc, 64, 64), 1, z(1, Cc, 64, 64),
                                      z(1, Cc, 64, 64), z(1), z(1, Cc))


def col2im_actbwd(k):
    return lambda o: o.col2im_actbwd(z(4, k * k * 4), 2, 2, k, z(1, 2 + k, 2 + k, 4), z(4), z(1, 2 + k, 2 + k, 4))


def gae(H, Md=4):
    J = H + 1
    return lambda o: o.gae_critic(H, Md, 0.99, 0.95, z(J * Md, 1), z(J * Md, 1), z(J * Md, 1), z(J * Md, 1), z(J, Md),
                                  z(H, Md), z(H, Md), z(H, Md), z(H, Md), z(H * Md, 1), z(8, dtype=torch.float64))


def actor_onehot(A, rows=8):
    acts = lambda: torch.nn.functional.one_hot(torch.zeros(rows, dtype=torch.long), A).float().to(DEV)
    return lambda o: o.actor_loss_onehot(1e-3, z(rows, A), acts(), z(rows), one(rows), z(rows, A), z(2, dtype=torch.float64))


def gather(N, ldw=None):
    ldw = ldw or N
    return lambda o: o.gather_rows(z(8, dtype=torch.int32), z(5, ldw)[:, :N], z(8, N))


# name: (a call just inside the boundary, the same call just outside it)
CASES = {
    "gemm_f16_lda_mod8": (f16_gemm(lda=72), f16_gemm(lda=68)),
    "gemm_f16_ldb_mod8": (f16_gemm(ldb=72), f16_gemm(ldb=68)),
    "gemm_f16_N_ge_8": (f16_gemm(N=8), f16_gemm(N=7)),
    "gemm_f16_K_ge_8": (f16_gemm(K=8, lda=8, ldb=8), f16_gemm(K=7, lda=8, ldb=8)),
    "gemm_f16_A_16_byte_aligned": (f16_gemm(lda=80, a_off=8), f16_gemm(lda=80, a_off=4)),
    "gemm_accumulate_no_bias": (lambda o: o.gemm(z(64, 64), z(64, 64), z(64, 64), accumulate=True),
                                lambda o: o.gemm(z(64, 64), z(64, 64), z(64, 64), bias=z(64), accumulate=True)),
    "conv_gemm_C_mod4": (conv(C=4), conv(C=6)),
    "conv_gemm_ldo_mod4": (conv(ldo=68), conv(ldo=66)),
    "ln_elu_fwd_N_le_1024": (ln_fwd(1024), ln_fwd(1025)),
    "ln_elu_bwd_N_le_1024": (ln_bwd(1024), ln_bwd(1025)),
    "cat_sample_C_le_32": (lambda o: o.cat_sample(z(4, 32), one(4, 32), 1, 32, z(4, 32)),
                           lambda o: o.cat_sample(z(4, 33), one(4, 33), 1, 33, z(4, 33))),
    "cat_st_bwd_C_le_32": (lambda o: o.cat_st_bwd(z(4, 32), 1, 32, z(4, 32), None, None, None, None, 0.0, z(4, 32)),
                           lambda o: o.cat_st_bwd(z(4, 33), 1, 33, z(4, 33), None, None, None, None, 0.0, z(4, 33))),
    "kl_G_le_32": (kl(32, 2), kl(33, 2)),
    "kl_C_le_32": (kl(2, 32), kl(2, 33)),
    "col2im_imgloss_channels_le_16": (imgloss(16), imgloss(17)),
    "col2im_actbwd_k_le_6": (col2im_actbwd(6), col2im_actbwd(7)),
    "im2col_input_ge_kernel": (lambda o: o.im2col(z(1, 4, 4, 4), 4, 0, z(1, 64)),
                               lambda o: o.im2col(z(1, 3, 3, 4), 4, 0, z(0, 64))),
    "colmean_N_le_32": (lambda o: o.colmean(z(4, 32), z(32)), lambda o: o.colmean(z(4, 33), z(33))),
    "gae_critic_H_le_127": (gae(127), gae(128)),
    "actor_loss_onehot_A_le_32": (actor_onehot(32), actor_onehot(33)),
    "gather_rows_N_mod4": (gather(8), gather(6)),
    "gather_rows_ldw_mod4": (gather(8, 12), gather(8, 10)),
    "vec_head_loss_K_le_4096": (lambda o: o.vec_head_loss(z(4, 4096), z(4, 4096), 1, z(4), z(4, 4096)),
                                lambda o: o.vec_head_loss(z(4, 4097), z(4, 4097), 1, z(4), z(4, 4097))),
}


@pytest.mark.parametrize("what", list(CASES))
def test_reference_table_accepts_and_refuses_what_the_native_table_does(native_ops, what):
    inside, outside = CASES[what]
    ref = VecRefOps(DEV)
    inside(native_ops)                            # accepted by both tables
    inside(ref)
    torch.cuda.synchronize()
    refused(native_ops, lambda: outside(native_ops))
    with pytest.raises(RuntimeError, match="unsupported"):
        outside(ref)
