"""CPU: the C-ABI library loads without a GPU and exports every symbol include/fvb200.h declares."""
import ctypes
import os
import re

from conftest import ROOT


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "fvb200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(fvb_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_entry_points():
    syms = declared_symbols()
    assert "fvb_linear_bf16" in syms and "fvb_attention_fwd" in syms and len(syms) >= 10


def test_library_exports_all_declared_symbols():
    from fastvideo_b200._lib import lib
    L = lib()
    missing = [s for s in declared_symbols() if not hasattr(L, s)]
    assert not missing, missing
    assert L.fvb_abi_version() == 2


def test_no_cpu_fallback_in_product_path():
    """The product path must fail loudly without CUDA tensors instead of silently computing on the CPU."""
    import pytest
    import torch
    from fastvideo_b200 import ops
    x = torch.zeros(8, 64, dtype=torch.bfloat16)
    with pytest.raises(ops.FvbError):
        ops.linear(x, x)


def test_product_never_imports_oracle():
    """oracle/ is test infrastructure: nothing under fastvideo_b200/ may import it."""
    pkg = os.path.join(ROOT, "fastvideo_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert "/root/reference" not in src, f


def test_plugin_routes_only_on_compute_capability_9_0(monkeypatch):
    """The library holds sm_90a code: the plug-in points route to it on a (9, 0) device and on nothing else."""
    import torch
    from fastvideo_b200 import plugin
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    for cap, want in (((9, 0), True), ((10, 0), False), ((8, 0), False), ((9, 1), False)):
        monkeypatch.setattr(torch.cuda, "get_device_capability", lambda *a, cap=cap: cap)
        assert plugin.device_supported() is want, cap
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    assert plugin.device_supported() is False
