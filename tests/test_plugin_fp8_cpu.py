"""CPU (build container): the "fvb200_fp8" quantization config resolves through the reference's registry and its
LinearMethodBase creates the same bf16 weight a plain nn.Linear state dict loads into. Quantisation and the GEMM need the
GPU: on CPU tensors they raise FvbError. Skipped where the reference tree is absent, like test_plugin_cpu.py."""
import pytest
import torch

from oracle import ref_shim

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present (set FVB_REFERENCE_ROOT or stage oracle/_ref/reference_py)")


@pytest.fixture(scope="module")
def plugin():
    ref_shim.install()
    from fastvideo_b200 import plugin as p
    ns = p.install(force=True)
    yield p, ns
    p.uninstall()


def test_fp8_linear_method_behind_replicated_linear(plugin):
    p, ns = plugin
    from fastvideo.layers.linear import LinearMethodBase, ReplicatedLinear
    from fastvideo.layers.quantization import get_quantization_config
    from fastvideo_b200._lib import FvbError
    cfg_cls = get_quantization_config(p.QUANT_NAME_FP8)
    assert cfg_cls is ns.Fvb200Fp8Config and cfg_cls.get_min_capability() == 90 and cfg_cls().get_name() == "fvb200_fp8"
    lin = ReplicatedLinear(256, 384, bias=True, params_dtype=torch.bfloat16, quant_config=cfg_cls(), prefix="blocks.0.to_q")
    assert isinstance(lin.quant_method, ns.Fvb200Fp8LinearMethod) and isinstance(lin.quant_method, LinearMethodBase)
    assert tuple(lin.weight.shape) == (384, 256) and lin.weight.dtype == torch.bfloat16
    src = torch.nn.Linear(256, 384).to(torch.bfloat16)
    lin.load_state_dict(src.state_dict())
    assert torch.equal(lin.weight, src.weight)
    with pytest.raises(FvbError):
        lin.quant_method.process_weights_after_loading(lin)  # CPU weights: no CPU quantiser
    with pytest.raises(FvbError):
        lin(torch.zeros(2, 5, 256, dtype=torch.bfloat16))
