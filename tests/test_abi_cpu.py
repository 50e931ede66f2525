"""CPU: the C-ABI library builds for sm_90a, loads without a GPU and exports every symbol that
include/vampnet_b200.h declares (no compute calls)."""
import os
import re

import pytest


@pytest.fixture(scope="module")
def built():
    from vampnet_b200 import build
    return build.build()


def test_library_loads_and_exports_header_symbols(built):
    from vampnet_b200 import _lib
    L = _lib.lib()
    header_version = int(re.search(r"#define VNB_ABI_VERSION (\d+)", open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "include", "vampnet_b200.h")).read()).group(1))
    assert L.vnb_abi_version() == header_version == 2
    header = open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "include", "vampnet_b200.h")).read()
    declared = set(re.findall(r"\b(vnb_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    for name in declared:
        assert hasattr(L, name), f"{name} declared in the header but not exported"
    assert declared == set(_lib.exported_symbols()), declared ^ set(_lib.exported_symbols())


def test_sass_has_hopper_instructions(built):
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", built], capture_output=True, text=True).stdout
    # wgmma of the GEMM (64x256), codec convolution (64x128) and attention (64x64); TMA 2-D / 3-D loads and the
    # multicast load of the paired GEMM; mbarrier waits
    for mnemonic in ("HGMMA.64x256x16.F32.BF16", "HGMMA.64x128x16.F32.BF16", "HGMMA.64x64x16.F32.BF16", "UTMALDG.2D",
                     "UTMALDG.3D", "UTMALDG.2D.MULTICAST", "SYNCS.PHASECHK.TRANS64.TRYWAIT"):
        assert mnemonic in sass, mnemonic
    # attention's P.V: the A operand (P) comes from registers, not from shared memory
    assert re.search(r"HGMMA\.64x64x16\.F32\.BF16 R\d+, R\d+, gdesc", sass), "no register-A wgmma"


def test_no_product_import_of_oracle():
    root = os.path.join(os.path.dirname(os.path.dirname(__file__)), "vampnet_b200")
    for dp, _, files in os.walk(root):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b|from\s+\.+\s*import\s+oracle|importlib.*oracle",
                                     src, re.M), f"{f} imports the oracle"
                assert "oracle" not in src, f"{f} mentions the oracle"


def test_options_are_host_state_with_measured_defaults(built):
    """vnb_get_option / vnb_set_option are plain host state (no device call): every documented switch exists, the
    default is the MEASURED configuration (single-CTA GEMM tiles, faster than CTA pairs on H100); the round-1 experimental
    switches are gone; unknown names fail."""
    import ctypes as C
    import subprocess
    import sys
    code = """
import ctypes as C, sys
lib = C.CDLL(sys.argv[1])
lib.vnb_get_option.argtypes = [C.c_char_p, C.POINTER(C.c_int32)]
lib.vnb_set_option.argtypes = [C.c_char_p, C.c_int32]
lib.vnb_last_error.restype = C.c_char_p
out = {}
for name in (b"gemm_pair", b"fused_sampler"):
    v = C.c_int32(-7)
    assert lib.vnb_get_option(name, C.byref(v)) == 0, name
    out[name.decode()] = v.value
assert out == {"gemm_pair": 0, "fused_sampler": 1}, out
assert lib.vnb_set_option(b"gemm_pair", 1) == 0
v = C.c_int32()
lib.vnb_get_option(b"gemm_pair", C.byref(v)); assert v.value == 1
for gone in (b"resid_tma", b"pair_arrive_cta", b"attn_p_tmem", b"attn_v2"):   # round-1 experiments: measured, then removed
    assert lib.vnb_set_option(gone, 1) != 0
assert lib.vnb_set_option(b"nope", 1) != 0 and b"unknown option" in lib.vnb_last_error()
print("ok")
"""
    env = {k: v for k, v in os.environ.items() if not k.startswith("VNB_")}  # defaults, not the caller's overrides
    r = subprocess.run([sys.executable, "-c", code, built], capture_output=True, text=True, env=env)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr[-2000:]
