"""The C-ABI shared library loads on a GPU-less box and exports every symbol that
include/evo_b200.h declares (no compute calls here)."""
import ctypes
import os
import re

import pytest

from evo_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "evo_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = re.findall(r"\b(evo_[a-z0-9_]+)\s*\(", src)
    return sorted(set(names))


def test_library_is_built_in_tree():
    assert os.path.exists(_lib.LIB_PATH), "run `python -m evo_b200.build` (or __graft_entry__.build())"
    assert os.path.dirname(_lib.LIB_PATH) == os.path.join(ROOT, "evo_b200")


def test_every_declared_symbol_is_exported():
    names = header_functions()
    assert len(names) >= 18
    handle = ctypes.CDLL(_lib.LIB_PATH)
    missing = [n for n in names if not hasattr(handle, n)]
    assert not missing, f"declared in include/evo_b200.h but not exported: {missing}"


def test_binding_table_covers_the_header():
    assert sorted(_lib.SIGNATURES) == header_functions()


def test_loader_binds_and_reports_abi_version_2():
    lib = _lib.lib()
    assert lib.evo_abi_version() == 2
    assert lib.evo_last_error() is not None
    lib.evo_reset_launch_count()
    assert lib.evo_launch_count() == 0


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.EvoError, match="no CPU"):
        _lib.lib()


def test_sass_has_wgmma_and_tma():
    """Hopper-native evidence: HGMMA (wgmma.mma_async) and UTMALDG (TMA) in the sm_90a code."""
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "HGMMA.64x256x16.F32.BF16" in sass and "UTMALDG" in sass
    assert "HMMA.16816" not in sass     # no legacy mma.sync tensor path


def test_header_is_plain_c_and_a_c_host_binds_abi_version_2(tmp_path):
    """include/evo_b200.h is the boundary for ANY host: it must compile as C99 and as C++ on its own, and a C program that
    #includes it and dlopen()s the library must resolve every declared entry point and get answers from the two that need no
    GPU (no torch, no Python anywhere near this binding)."""
    import shutil
    import subprocess
    gcc, gxx = shutil.which("gcc"), shutil.which("g++")
    if not gcc or not gxx:
        pytest.skip("gcc / g++ not available")
    hdr = os.path.join(ROOT, "include", "evo_b200.h")
    for cmd in ([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-x", "c", hdr],
                [gxx, "-std=c++11", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-x", "c++", hdr]):
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    names = header_functions()
    src = tmp_path / "host.c"
    src.write_text(
        '#include <dlfcn.h>\n#include <stdio.h>\n#include "evo_b200.h"\n'
        "int main(int argc, char** argv) {\n"
        "  void* h = dlopen(argv[1], RTLD_NOW | RTLD_LOCAL);\n"
        '  if (!h) { fprintf(stderr, "dlopen: %s\\n", dlerror()); return 2; }\n'
        "  const char* names[] = {" + ", ".join(f'"{n}"' for n in names) + "};\n"
        "  int missing = 0;\n"
        "  for (unsigned i = 0; i < sizeof(names) / sizeof(names[0]); ++i) if (!dlsym(h, names[i])) { fprintf(stderr, \"missing %s\\n\", names[i]); ++missing; }\n"
        "  int (*version)(void) = (int (*)(void))dlsym(h, \"evo_abi_version\");\n"
        "  const char* (*last_error)(void) = (const char* (*)(void))dlsym(h, \"evo_last_error\");\n"
        '  printf("%d %d %s\\n", missing, version(), last_error() ? "str" : "null");\n'
        "  (void)argc; return missing != 0;\n}\n")
    exe = tmp_path / "host"
    r = subprocess.run([gcc, "-std=gnu99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-ldl"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe), _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.split() == ["0", "2", "str"], (r.stdout, r.stderr)


def test_error_convention_without_a_gpu():
    """No exception crosses the ABI: a rejected argument returns a negative code and leaves the reason in evo_last_error() before
    anything is launched (so this runs on a GPU-less box); and a well-formed call on a box without a GPU FAILS, loudly, with the
    CUDA runtime's reason -- there is no CPU path to fall back to."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("this is the GPU-less half of the error convention")
    lib = _lib.lib()
    p = _lib.GemmParams(A=0x1000, lda=100, W=0x2000, C=0x3000, ldc=64, bias=None, residual=None, ldr=64, M=4, N=64, K=100, epilogue=0, variant=0)
    assert lib.evo_gemm(ctypes.byref(p), None) < 0 and b"K (100) must be a multiple of 64" in lib.evo_last_error()
    p.K, p.N, p.variant = 128, 256, 4
    assert lib.evo_gemm(ctypes.byref(p), None) < 0 and b"evo_gemm: unknown variant 4" in lib.evo_last_error()
    s = _lib.GemmSmallMParams(A=0x1000, lda=64, W=0x2000, C=0x3000, ldc=256, M=4, N=256, K=64, epilogue=7)
    assert lib.evo_gemm_smallm(ctypes.byref(s), None) < 0 and b"evo_gemm_smallm: unknown epilogue 7" in lib.evo_last_error()
    assert lib.evo_sample(None, None, 2, 2000, 1, 0.0, 1.0, 0, 0, None) < 0 and b"vocabulary 2000 unsupported" in lib.evo_last_error()
    assert lib.evo_kv_append(None, None, 1, 10, 2, 128, 10, 16, None) < 0 and b"exceeds the KV cache (16)" in lib.evo_last_error()   # mha.py:367
    with pytest.raises(_lib.EvoError, match="exceeds the KV cache"):
        _lib.check(lib.evo_kv_append(None, None, 1, 10, 2, 128, 10, 16, None), "evo_kv_append")
    rc = lib.evo_rmsnorm(ctypes.c_void_p(0x1000), ctypes.c_void_p(0x2000), ctypes.c_void_p(0x3000), 4, 4096, 1e-6, None)
    assert rc < 0 and b"failed" in lib.evo_last_error()

    # packed forms: bad geometry is rejected with its reason before anything touches the device (a workspace query answers 0)
    def hyena(**kw):
        f = dict(z=0x1000, y=0x2000, cu_seqlens=0x3000, n_seq=1, T=256, max_seqlen=256, D=256, S=8, nheads=2)
        f.update(kw)
        return _lib.HyenaVarlenParams(**f)

    def rejected(rc, msg):
        return rc < 0 and msg in lib.evo_last_error()

    def ws_rejected(n, msg):
        return n == 0 and msg in lib.evo_last_error()

    no_cu = b"needs cu_seqlens and 0 < max_seqlen <= T < 2^31"
    p = hyena(cu_seqlens=None)
    assert rejected(lib.evo_hyena_fwd_varlen(ctypes.byref(p), None, 0, None), no_cu)
    p = hyena(max_seqlen=300)
    assert ws_rejected(lib.evo_hyena_fwd_varlen_workspace(ctypes.byref(p)), b"(max_seqlen 300, T 256)")
    p = hyena(nheads=4)
    assert rejected(lib.evo_hyena_fwd_varlen(ctypes.byref(p), None, 0, None), b"needs head_dim 128 and D % 256 == 0 (D 256, 4 heads)")
    c = _lib.HyenaVarlenCkptParams(base=hyena(cu_seqlens=None))
    assert rejected(lib.evo_hyena_fwd_varlen_ckpt(ctypes.byref(c), None, 0, None), no_cu)
    c = _lib.HyenaVarlenCkptParams(base=hyena(max_seqlen=301))
    assert ws_rejected(lib.evo_hyena_fwd_varlen_ckpt_workspace(ctypes.byref(c)), b"(max_seqlen 301, T 256)")
    c = _lib.HyenaVarlenCkptParams(base=hyena(), ckpt_states=0x4000, ckpt_base=0x5000, ckpt_stride=100, n_ckpt=4)
    assert rejected(lib.evo_hyena_fwd_varlen_ckpt(ctypes.byref(c), None, 0, None),
                    b"evo_hyena_fwd_varlen_ckpt: checkpoints need ckpt_base, n_ckpt > 0 and a stride that is a positive multiple of 128 (got 100)")
    c.ckpt_stride = 228
    assert ws_rejected(lib.evo_hyena_fwd_varlen_ckpt_workspace(ctypes.byref(c)), b"multiple of 128 (got 228)")

    a = _lib.AttnVarlenParams(q=0x1000, k=0x2000, v=0x3000, out=0x4000, q_tok_stride=384, kv_tok_stride=384, cu_seqlens=None, n_seq=1,
                              T=256, max_seqlen=256, H=1, hd=128, softmax_scale=0.088)
    assert rejected(lib.evo_attn_fwd_varlen(ctypes.byref(a), None), b"evo_attn_fwd_varlen: " + no_cu)
    a.cu_seqlens, a.max_seqlen = 0x5000, 257
    assert rejected(lib.evo_attn_fwd_varlen(ctypes.byref(a), None), b"(max_seqlen 257, T 256)")
    a.max_seqlen, a.hd = 256, 64
    assert rejected(lib.evo_attn_fwd_varlen(ctypes.byref(a), None), b"evo_attn_fwd_varlen: head_dim 64 unsupported")
    a = _lib.AttnVarlenPrefixParams(qkv=0x1000, out=0x2000, cu_seqlens=0x3000, n_seq=1, T=256, max_seqlen=256, cache=None, n_cache=1,
                                    cache_len=256, prefix_seq=0x4000, prefix_len=0x5000, H=1, hd=128, softmax_scale=0.088)
    assert rejected(lib.evo_attn_fwd_varlen_prefix(ctypes.byref(a), None), b"evo_attn_fwd_varlen_prefix: needs a cache")
    a.cu_seqlens = None
    assert rejected(lib.evo_attn_fwd_varlen_prefix(ctypes.byref(a), None), b"evo_attn_fwd_varlen_prefix: " + no_cu)
    a.cu_seqlens, a.hd = 0x3000, 96
    assert rejected(lib.evo_attn_fwd_varlen_prefix(ctypes.byref(a), None), b"evo_attn_fwd_varlen_prefix: head_dim 96 unsupported")
