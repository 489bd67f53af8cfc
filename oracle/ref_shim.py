"""TEST INFRASTRUCTURE ONLY -- makes the reference's own Python importable on a CPU-only box.

The reference tree is $FVB_REFERENCE_ROOT, else oracle/_ref/reference_py (staged by oracle/stage_ref_kernels.py,
git-ignored). oracle/gen_golden.py uses this to (a) validate the restatements in oracle/*.py against the reference itself
and (b) write the small golden fixtures under tests/golden/; tests/test_plugin_cpu.py uses it to register the plug-in into
the reference. Nothing on the product path, in smoke() or in bench.py's GPU arm imports it.

Recipe (SURVEY.md section 8c / Appendix A): register a bare `fastvideo` package whose __path__ points at
<reference root>/fastvideo (skipping fastvideo/__init__.py, which pulls in imageio/diffusers via
VideoGenerator), stub the three missing third-party roots, point the CPU platform at the SDPA backend
(fastvideo/platforms/interface.py:122-125 returns "" on CPU) and make get_local_torch_device() return
cpu (fastvideo/distributed/parallel_state.py:881-890 maps non-CUDA to mps).
"""
from __future__ import annotations

import importlib.abc
import importlib.machinery
import importlib.util
import os
import socket
import sys
import types

_HERE = os.path.dirname(os.path.abspath(__file__))
# the reference's Python: $FVB_REFERENCE_ROOT, else the copy oracle/stage_ref_kernels.py stages into oracle/_ref/reference_py
REF_ROOT = os.environ.get("FVB_REFERENCE_ROOT") or os.path.join(_HERE, "_ref", "reference_py")
_STUB_ROOTS = {"imageio", "diffusers", "remote_pdb"}
_installed = False


class _Stub(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return type(name, (), {})


class _Finder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, name, path, target=None):
        if name.split(".")[0] in _STUB_ROOTS:
            return importlib.machinery.ModuleSpec(name, self, is_package=True)
        # the staged copy of the reference (oracle/stage_ref_kernels.py) leaves out fastvideo/third_party (261 MB of
        # vendored eval / other-model code, none of it on the Wan path): stub it when it is not there
        if (name == "fastvideo.third_party" or name.startswith("fastvideo.third_party.")) and not os.path.isdir(
                os.path.join(REF_ROOT, "fastvideo", "third_party")):
            return importlib.machinery.ModuleSpec(name, self, is_package=True)
        return None

    def create_module(self, spec):
        m = _Stub(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        # Minimal working stand-ins for the few diffusers names the reference's SCHEDULERS need to run on CPU
        # (config registration, output containers); everything else stays an inert stub class.
        fill = _DIFFUSERS_EMULATION.get(module.__name__)
        if fill is not None:
            for k, v in fill().items():
                setattr(module, k, v)


def _emulate_configuration_utils():
    import functools
    import inspect

    class ConfigMixin:
        config_name = None

        def register_to_config(self, **kwargs):
            d = dict(vars(getattr(self, "_internal_dict", types.SimpleNamespace())))
            d.update(kwargs)
            self._internal_dict = types.SimpleNamespace(**d)

        @property
        def config(self):
            return self._internal_dict

    def register_to_config(init):
        @functools.wraps(init)
        def inner(self, *args, **kwargs):
            sig = inspect.signature(init)
            bound = sig.bind(self, *args, **kwargs)
            bound.apply_defaults()
            cfg = {k: v for k, v in bound.arguments.items() if k not in ("self", "kwargs")}
            cfg.update(bound.arguments.get("kwargs", {}))
            self._internal_dict = types.SimpleNamespace(**cfg)
            init(self, *args, **kwargs)
        return inner

    return dict(ConfigMixin=ConfigMixin, register_to_config=register_to_config)


def _emulate_scheduling_utils():
    import enum
    from dataclasses import dataclass

    class KarrasDiffusionSchedulers(enum.Enum):
        UniPCMultistepScheduler = 1

    class SchedulerMixin:
        pass

    @dataclass
    class SchedulerOutput:
        prev_sample: object = None

    return dict(KarrasDiffusionSchedulers=KarrasDiffusionSchedulers, SchedulerMixin=SchedulerMixin, SchedulerOutput=SchedulerOutput)


def _emulate_utils():
    class BaseOutput:
        pass

    return dict(BaseOutput=BaseOutput, deprecate=lambda *a, **k: None)


_DIFFUSERS_EMULATION = {"diffusers.configuration_utils": _emulate_configuration_utils,
                        "diffusers.schedulers.scheduling_utils": _emulate_scheduling_utils,
                        "diffusers.utils": _emulate_utils}


def available() -> bool:
    return os.path.isdir(os.path.join(REF_ROOT, "fastvideo"))


def install() -> None:
    """Idempotent. After this, `import fastvideo.<submodule>` resolves into the reference tree."""
    global _installed
    if _installed:
        return
    if not available():
        raise RuntimeError(f"reference tree not found at {REF_ROOT}")
    import torch

    pkg = types.ModuleType("fastvideo")
    pkg.__path__ = [os.path.join(REF_ROOT, "fastvideo")]
    pkg.__spec__ = importlib.machinery.ModuleSpec("fastvideo", None, is_package=True)
    pkg.__spec__.submodule_search_locations = pkg.__path__
    sys.modules["fastvideo"] = pkg
    sys.meta_path.insert(0, _Finder())

    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    if "MASTER_PORT" not in os.environ:
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        os.environ["MASTER_PORT"] = str(s.getsockname()[1])
        s.close()

    from fastvideo.platforms.cpu import CpuPlatform
    CpuPlatform.get_attn_backend_cls = classmethod(
        lambda cls, sel, head_size, dtype: "fastvideo.attention.backends.sdpa.SDPABackend")
    # The shim is the reference's CPU path by definition. On a box that HAS a GPU (bench.py's CPU arm on the GPU host)
    # the reference would resolve CudaPlatform through NVML (fastvideo/platforms/__init__.py:16-49); pin the CPU platform.
    import fastvideo.platforms as _plat
    if not isinstance(getattr(_plat, "_current_platform", None), CpuPlatform):
        _plat._current_platform = CpuPlatform()
    import fastvideo.distributed.parallel_state as ps
    ps.get_local_torch_device = lambda: torch.device("cpu")
    ps.maybe_init_distributed_environment_and_model_parallel(1, 1)
    _installed = True


def load_kernel_pkg_module(rel: str, name: str):
    """Load one file of fastvideo-kernel/python/fastvideo_kernel by path (the package __init__ imports
    Triton kernels that query a GPU driver at import time: triton_kernels/st_attn_triton.py:7-49)."""
    path = os.path.join(REF_ROOT, "fastvideo-kernel", "python", "fastvideo_kernel", rel)
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod
