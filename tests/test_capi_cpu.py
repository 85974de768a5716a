"""CPU: the C-ABI library builds for sm_90a, loads without a GPU, and exports exactly what
include/moshi_b200.h declares.  No compute entry point is called here."""
import ctypes as C
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def built():
    from moshi_b200.build import build
    return build()


def _declared() -> set[str]:
    text = (ROOT / "include" / "moshi_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", text))


def test_header_and_library_agree(built):
    from moshi_b200 import _lib
    declared = _declared()
    assert len(declared) >= 40
    lib = C.CDLL(str(built))
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, f"declared in moshi_b200.h but not exported: {missing}"
    assert declared == set(_lib.EXPORTED_SYMBOLS), declared ^ set(_lib.EXPORTED_SYMBOLS)


def test_library_reports_version_and_errors_without_gpu(built):
    from moshi_b200 import _lib
    lib = _lib.lib()
    assert lib.b200_abi_version() == _lib.ABI_VERSION == 2
    assert lib.b200_launch_count() == 0
    cfg = _lib.MimiConfigC()          # all zero: invalid
    h = C.c_void_p()
    rc = lib.b200_mimi_create(C.byref(cfg), C.byref(h))
    assert rc == _lib.B200_ERR_INVALID
    assert b"n_ratios" in lib.b200_last_error()
    with pytest.raises(ValueError):
        _lib.check(rc)
    lcfg = _lib.LMConfigC()
    rc = lib.b200_lm_create(C.byref(lcfg), C.byref(h))
    assert rc == _lib.B200_ERR_INVALID


def test_sass_is_sm100a_only(built):
    """The library carries SASS for sm_90a (H100) and nothing else.  The name predates the move from sm_100a and is kept so
    that the test keeps its id from run to run."""
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-lelf", str(built)], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_product_does_not_import_oracle():
    bad = []
    for p in (ROOT / "moshi_b200").rglob("*.py"):
        src = p.read_text()
        if re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M):
            bad.append(str(p))
    assert not bad, f"product code must not depend on the oracle: {bad}"
