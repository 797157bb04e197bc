"""CPU: the C-ABI library builds for sm_90a, loads, and exports every symbol that
include/envpool_b200.h declares.  No compute calls (no GPU here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_engine_exports_every_declared_symbol_at_abi_version_3(engine_built):
    """Version 3: a NaN HalfCheetah weight or noise scale in epb_config selects the default, and
    every other value, negative included, is used as given (up to version 2 any negative value
    selected the default).  The header, the library and the pybind modules must agree on it."""
    from envpool_b200 import _capi
    from envpool_b200.classic_control import classic_control_envpool

    hdr = open(os.path.join(ROOT, "include", "envpool_b200.h")).read()
    declared = set(re.findall(r"\b(epb_[a-z_0-9]+)\s*\(", hdr))
    declared -= {"epb_pool"}
    assert declared == set(_capi.ABI_SYMBOLS), declared ^ set(_capi.ABI_SYMBOLS)
    lib = ctypes.CDLL(_capi.ENGINE_SO)
    for sym in sorted(declared):
        assert hasattr(lib, sym), f"missing export {sym}"
    assert lib.epb_abi_version() == 3
    assert re.search(r"#define EPB_ABI_VERSION (\d+)", hdr).group(1) == "3"
    assert classic_control_envpool.__abi_version__ == 3


def test_engine_is_sm_90a_sass():
    import shutil
    import subprocess

    from envpool_b200 import _capi

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-lelf", _capi.ENGINE_SO], capture_output=True,
                         text=True).stdout
    assert "sm_90a" in out, out


def test_product_never_touches_the_oracle():
    """The shipped package must not import, link, call or even name anything under oracle/."""
    pkg = os.path.join(ROOT, "envpool_b200")
    offenders = []
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cc", ".h")):
                text = open(os.path.join(dirpath, f), errors="ignore").read().lower()
                if "oracle" in text:
                    offenders.append(os.path.join(dirpath, f))
    hdr = open(os.path.join(ROOT, "include", "envpool_b200.h")).read().lower()
    if "oracle" in hdr:
        offenders.append("include/envpool_b200.h")
    assert not offenders, offenders


def test_create_fails_loudly_without_gpu(engine_built):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from envpool_b200 import _capi

    with pytest.raises((_capi.EpbError, ValueError)):
        _capi.CPool("CartPole", 8)
