"""not gpu: the C-ABI library loads on a CPU-only host and exports every symbol include/*.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "meshanything_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ma_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_entry_points():
    names = _declared()
    for must in ("ma_decode_generate", "ma_linear_f16", "ma_attention_f16", "ma_layernorm", "ma_last_error"):
        assert must in names


def test_library_loads_and_exports_all_symbols():
    from meshanything_b200 import capi
    lib = capi.lib()
    assert lib.ma_abi_version() == 1
    raw = ctypes.CDLL(capi.lib_path())
    for name in _declared():
        assert hasattr(raw, name), f"{name} declared in the header but not exported"
    assert set(capi.EXPORTS) <= set(_declared())


def test_size_queries_need_no_gpu():
    from meshanything_b200 import capi
    lib = capi.lib()
    # 24 layers x K,V x 16 heads x 64 x fp16 = 98304 bytes per cached position (SURVEY.md 8d)
    assert lib.ma_kv_cache_bytes(24, 1, 1000) == 98304 * 1000
    assert lib.ma_kv_cache_bytes(24, 64, 7459) == 98304 * 7459 * 64
    assert lib.ma_decoder_workspace_bytes(1, 7459) > 0
    assert lib.ma_attention_scratch_bytes(1, 16, 7459) > 0


def test_product_does_not_import_the_oracle():
    """The product packages must not reference oracle/ (it is test infrastructure)."""
    bad = []
    for pkg in ("meshanything_b200", "MeshAnything"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, pkg)):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".h")):
                    txt = open(os.path.join(dirpath, f)).read()
                    if re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M) or "libma_oracle" in txt:
                        bad.append(os.path.join(dirpath, f))
    assert not bad, bad


def test_library_targets_sm90a_and_uses_wgmma():
    """The library is compiled for the H100 (sm_90a) only, and the tensor-core kernels (gemm_tc, gemm_ws, attention_tc)
    run on wgmma (SASS HGMMA) fed by TMA (UTMALDG)."""
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        import pytest
        pytest.skip("cuobjdump not available")
    from meshanything_b200 import capi
    capi.lib()
    sass = subprocess.run([cuobjdump, "-sass", capi.lib_path()], capture_output=True, text=True, timeout=600).stdout
    archs = set(re.findall(r"arch = (sm_\w+)", sass))
    assert archs == {"sm_90a"}, archs
    assert "HGMMA" in sass and "UTMALDG" in sass


def _prototypes():
    """{name: number of parameters} for every function the header declares (void parameter lists count 0)."""
    src = open(os.path.join(ROOT, "include", "meshanything_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    out = {}
    for m in re.finditer(r"\b(ma_[a-z0-9_]+)\s*\(([^;{}]*?)\)\s*;", src, flags=re.S):
        params = m.group(2).strip()
        out[m.group(1)] = 0 if params in ("", "void") else params.count(",") + 1
    return out


def test_ctypes_signatures_match_the_header():
    """Every entry point for which capi.py sets `argtypes` must take exactly as many arguments as the header's prototype:
    a ctypes call with a stale signature corrupts the stack silently instead of failing."""
    from meshanything_b200 import capi
    lib = capi.lib()
    protos = _prototypes()
    assert set(_declared()) <= set(protos), sorted(set(_declared()) - set(protos))
    checked = 0
    for name, n in protos.items():
        fn = getattr(lib, name)
        if fn.argtypes is not None:
            assert len(fn.argtypes) == n, f"{name}: header has {n} parameters, capi.py declares {len(fn.argtypes)}"
            checked += 1
    assert checked >= 25, checked
