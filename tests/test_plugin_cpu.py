"""CPU (build container): fastvideo_b200.plugin registers REAL subclasses behind the reference's plug-in points.

Runs the reference's own selector / registry / module constructors (imported through oracle/ref_shim) and checks that
they resolve to the libfvb200 classes, that the ABC contracts hold (the classes instantiate), that a reference
`ReplicatedLinear` accepts the LinearMethodBase, and that a reference WanTransformerBlock's state_dict() loads into
wan_dit.WanBlock. No compute is run (no GPU here): with CPU tensors the ops raise FvbError, which is asserted too.
Skipped where the reference tree is absent ($FVB_REFERENCE_ROOT, else oracle/_ref/reference_py).
"""
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


def test_dense_backend_resolves_through_the_reference_selector(plugin):
    p, ns = plugin
    from fastvideo.attention.backends.abstract import AttentionBackend, AttentionImpl, AttentionMetadata, AttentionMetadataBuilder
    from fastvideo.attention.selector import backend_name_to_enum, get_attn_backend
    from fastvideo.platforms.interface import AttentionBackendEnum as E
    supported = (E.FLASH_ATTN, E.TORCH_SDPA)
    be = get_attn_backend(128, torch.bfloat16, supported_attention_backends=supported)
    assert be is ns.Fvb200AttentionBackend and issubclass(be, AttentionBackend)
    # distinct name, and the name resolves to an enum member (attention/layer.py:78)
    assert be.get_name() == p.DENSE_BACKEND_NAME != "TORCH_SDPA"
    assert backend_name_to_enum(be.get_name()) is E[p.DENSE_BACKEND_NAME]
    impl = be.get_impl_cls()(num_heads=4, head_size=128, softmax_scale=128 ** -0.5, causal=False, num_kv_heads=4, prefix="x.impl")
    assert isinstance(impl, AttentionImpl)
    md = be.get_builder_cls()().build(current_timestep=3)
    assert isinstance(md, AttentionMetadata) and isinstance(md, be.get_metadata_cls()) and md.current_timestep == 3
    assert isinstance(be.get_builder_cls()(), AttentionMetadataBuilder)
    q = torch.zeros(1, 64, 4, 128, dtype=torch.bfloat16)
    with pytest.raises(Exception) as ei:  # no CPU fallback
        impl.forward(q, q, q, md)
    assert "Fvb" in type(ei.value).__name__ or "CUDA" in str(ei.value) or "cuda" in str(ei.value)
    # fp32 / other head sizes keep the reference's own table (CPU shim: SDPA)
    other = get_attn_backend(64, torch.float32, supported_attention_backends=supported)
    assert other.__name__ == "SDPABackend"


def test_vsa_backend_keeps_class_identity_and_swaps_the_impl(plugin):
    p, ns = plugin
    from fastvideo.attention.backends.abstract import AttentionImpl
    from fastvideo.attention.backends import video_sparse_attn as V
    B = V.VideoSparseAttentionBackend
    assert B.get_name() == "VIDEO_SPARSE_ATTN"          # wanvideo.py:628-629 / denoising.py:466 keep working
    assert B.get_impl_cls() is ns.Fvb200VideoSparseAttentionImpl
    assert issubclass(B.get_impl_cls(), V.VideoSparseAttentionImpl) and issubclass(B.get_impl_cls(), AttentionImpl)
    assert issubclass(B.get_builder_cls(), V.VideoSparseAttentionMetadataBuilder)
    assert issubclass(B.get_metadata_cls(), V.VideoSparseAttentionMetadata)
    impl = B.get_impl_cls()(num_heads=2, head_size=128, causal=False, softmax_scale=128 ** -0.5, prefix="blocks.0.attn.impl")
    assert hasattr(impl, "preprocess_qkv") and hasattr(impl, "postprocess_output")
    # the metadata class carries every field of the reference's dataclass
    import dataclasses
    ref_fields = {f.name for f in dataclasses.fields(V.VideoSparseAttentionMetadata)}
    assert ref_fields <= {f.name for f in dataclasses.fields(B.get_metadata_cls())}


def test_linear_method_behind_replicated_linear(plugin):
    p, ns = plugin
    from fastvideo.layers.linear import LinearMethodBase, ReplicatedLinear
    from fastvideo.layers.quantization import get_quantization_config
    cfg_cls = get_quantization_config(p.QUANT_NAME)
    assert cfg_cls is ns.Fvb200Bf16Config
    lin = ReplicatedLinear(256, 384, bias=True, params_dtype=torch.bfloat16, quant_config=cfg_cls(), prefix="blocks.0.to_q")
    assert isinstance(lin.quant_method, ns.Fvb200LinearMethod) and isinstance(lin.quant_method, LinearMethodBase)
    assert tuple(lin.weight.shape) == (384, 256) and lin.weight.dtype == torch.bfloat16
    # a plain nn.Linear state dict loads (same parameter names / layout as UnquantizedLinearMethod)
    src = torch.nn.Linear(256, 384).to(torch.bfloat16)
    lin.load_state_dict(src.state_dict())
    assert torch.equal(lin.weight, src.weight)
    from fastvideo_b200._lib import FvbError
    with pytest.raises(FvbError):
        lin(torch.zeros(2, 5, 256, dtype=torch.bfloat16))


def test_rmsnorm_custom_op_dispatches_to_forward_cuda_only_with_a_gpu(plugin):
    p, ns = plugin
    from fastvideo.layers.custom_op import CustomOp
    from fastvideo.layers.layernorm import RMSNorm
    n = RMSNorm(256, eps=1e-6)
    assert RMSNorm.__dict__["forward_cuda"] is p.rms_norm_forward_cuda
    assert CustomOp.op_registry["rms_norm"] is RMSNorm
    # no GPU in this container: dispatch stays on forward_native (and therefore still computes)
    assert n._forward_method.__func__ is RMSNorm.forward_native
    x = torch.randn(2, 3, 256)
    assert torch.allclose(n(x), x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6), atol=1e-6)


def test_reference_block_state_dict_loads_into_wanblock(plugin):
    p, ns = plugin
    from fastvideo.models.dits.wanvideo import WanTransformerBlock
    from fastvideo.platforms.interface import AttentionBackendEnum as E
    blk = WanTransformerBlock(256, 512, 2, "rms_norm_across_heads", True, 1e-6, None, (E.TORCH_SDPA,), prefix="blocks.0")
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():  # the reference allocates weights with torch.empty
        for prm in blk.parameters():
            prm.copy_(torch.randn(prm.shape, generator=g))
    ours = p.load_wan_block(blk)
    sd = blk.state_dict()
    assert tuple(ours.w_qkv.shape) == (3 * 256, 256)
    assert torch.equal(ours.w_qkv[:256], sd["to_q.weight"].to(torch.bfloat16))
    assert torch.equal(ours.w_1, sd["ffn.fc_in.weight"].to(torch.bfloat16))
    assert torch.equal(ours.scale_shift_table, sd["scale_shift_table"])


def test_uninstall_restores_the_reference(plugin):
    p, ns = plugin
    from fastvideo.attention.backends import video_sparse_attn as V
    p.uninstall()
    try:
        assert V.VideoSparseAttentionBackend.get_impl_cls() is V.VideoSparseAttentionImpl
        from fastvideo.layers.layernorm import RMSNorm
        assert "forward_cuda" not in RMSNorm.__dict__
    finally:
        p.install(force=True)
