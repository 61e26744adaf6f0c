"""CPU-side checks of the C ABI: the library builds/loads here (nvcc cross-compiles, no GPU needed)
and exports every symbol include/pd_b200.h declares.  No compute calls."""
import ctypes
import subprocess

from pydreamer_b200 import _native


def test_header_parses_all_entry_points():
    protos = _native.parse_header()
    assert len(protos) >= 39
    for must in ("pd_create", "pd_gemm", "pd_ln_elu_fwd", "pd_gru_bwd", "pd_cat_sample", "pd_kl", "pd_im2col",
                 "pd_col2im_imgloss", "pd_gae_critic", "pd_adamw"):
        assert must in protos
    assert len(protos["pd_gemm"][1]) == 21


def test_library_exports_every_declared_symbol():
    lib = _native.load()
    out = subprocess.run(["nm", "-D", "--defined-only", _native.LIB_PATH], capture_output=True, text=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    for name in _native.parse_header():
        assert name in exported, f"{name} declared in pd_b200.h but not exported"
        assert hasattr(lib, name)


def test_version_and_error_paths_without_gpu():
    lib = _native.load()
    assert b"sm_90a" in lib.pd_version()
    h = ctypes.c_void_p()
    rc = lib.pd_create(0, ctypes.byref(h))
    # no GPU in the authoring container: must fail cleanly, never fall back
    if rc != 0:
        assert not h.value
    else:
        lib.pd_destroy(h)


def test_sass_contains_hopper_tensor_and_tma_instructions():
    sass = subprocess.run(["cuobjdump", "-sass", _native.LIB_PATH], capture_output=True, text=True).stdout
    assert "HGMMA.64x128x8.F32.TF32" in sass         # wgmma tf32 (K-major operands)
    assert "HGMMA.64x128x16.F32" in sass             # wgmma fp16
    assert "HMMA.1688.F32.TF32" in sass              # mma.sync tf32 (MN-major operands)
    assert "UTMALDG" in sass                         # TMA tensor load
    assert "UTMASTG" in sass and "UTMAREDG" in sass  # TMA tensor store / reduce-add epilogues
    assert "UTMALDG.4D.IM2COL" in sass               # implicit-GEMM convolution operands


import pytest


@pytest.mark.parametrize("cname,pyname", (("pd_rssm_fwd_args", "RssmFwdArgs"), ("pd_rssm_bwd_args", "RssmBwdArgs")))
def test_struct_argument_layout_matches_the_header(tmp_path, cname, pyname):
    """The two argument structs of the ABI: the ctypes mirrors (ops.RssmFwdArgs / ops.RssmBwdArgs) must have the C
    compiler's size and field offsets for the declarations in include/pd_b200.h."""
    import os

    from pydreamer_b200 import ops as _ops_mod

    RssmFwdArgs = getattr(_ops_mod, pyname)
    fields = [n for n, _ in RssmFwdArgs._fields_]
    src = tmp_path / "layout.c"
    body = "".join(f'    printf("{n} %zu\\n", offsetof({cname}, {n}));\n' for n in fields)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pd_b200.h"\nint main(void) {\n'
                   f'    printf("sizeof %zu\\n", sizeof({cname}));\n' + body + "    return 0;\n}\n")
    exe = tmp_path / "layout"
    inc = os.path.join(os.path.dirname(os.path.abspath(_native.HEADER)))
    subprocess.run(["gcc", "-I", inc, str(src), "-o", str(exe)], check=True)       # the header is plain C
    out = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out.pop("sizeof")) == ctypes.sizeof(RssmFwdArgs)
    assert list(out) == fields                                                      # same fields, same order
    for n in fields:
        assert int(out[n]) == getattr(RssmFwdArgs, n).offset, n


def test_sass_of_the_persistent_bptt_kernel():
    sass = subprocess.run(["cuobjdump", "-sass", "-fun", "rssm_unroll_bwd_kernel", _native.LIB_PATH],
                          capture_output=True, text=True).stdout
    if "HMMA" not in sass:
        sass = subprocess.run(["cuobjdump", "-sass", _native.LIB_PATH], capture_output=True, text=True).stdout
    assert "UTMALDG.2D" in sass                  # operands staged by TMA (cp.async.bulk.tensor.2d)
    assert "HMMA.1688.F32.TF32" in sass          # mma.sync.m16n8k8 tf32
    assert "SYNCS" in sass and "LDSM" in sass    # mbarrier pipeline, ldmatrix weight fragments


def test_sass_of_the_persistent_rssm_kernel():
    sass = subprocess.run(["cuobjdump", "-sass", "-fun", "rssm_unroll_fwd3_kernel", _native.LIB_PATH],
                          capture_output=True, text=True).stdout
    if "HMMA" not in sass:                       # older cuobjdump: -fun wants the mangled name; fall back to the whole file
        sass = subprocess.run(["cuobjdump", "-sass", _native.LIB_PATH], capture_output=True, text=True).stdout
    assert "UTMALDG.2D" in sass                  # TMA tile staging
    assert "SYNCS" in sass                       # mbarrier pipeline
    assert "HMMA.16816.F32" in sass and "LDSM" in sass   # mma.sync m16n8k16 + ldmatrix contractions
