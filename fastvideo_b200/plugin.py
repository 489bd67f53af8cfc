"""Registration of libfvb200 behind FastVideo's own plug-in points -- real subclasses of the reference's ABCs, created
and registered when (and only when) the `fastvideo` package is importable.

    import fastvideo_b200.plugin as fvb_plugin
    fvb_plugin.install()          # in the process that runs FastVideo, before the model is built

What install() registers, and the reference interface each piece stands behind:

  attention (dense)   Fvb200AttentionBackend / Impl / Metadata / MetadataBuilder subclass
                      fastvideo/attention/backends/abstract.py:31-194. The platform's backend table
                      (fastvideo/platforms/cuda.py:111-288 `get_attn_backend_cls`) is wrapped so that bf16, head_size 128
                      requests for FLASH_ATTN / TORCH_SDPA / "no preference" resolve to it; its get_name() is the distinct
                      "FVB200_ATTN", added to AttentionBackendEnum (fastvideo/platforms/interface.py:13-27) so that
                      `backend_name_to_enum(get_name())` (fastvideo/attention/layer.py:78) resolves.
  attention (8-bit)   Fvb200Attention8bitBackend / Impl: the same contract on the 8-bit attention (INT8 Q K^T, FP8 P V,
                      ops.attention_8bit), under its own enum member "FVB200_ATTN_8BIT". Only an explicit selection of that
                      name resolves to it (same bf16 / head_size 128 / sm_90 rules); the reference's SAGE_ATTN is untouched.
  attention (VSA)     Fvb200VideoSparseAttentionImpl / MetadataBuilder / Metadata subclass the classes in
                      fastvideo/attention/backends/video_sparse_attn.py:115-342 and are returned by the reference's OWN
                      `VideoSparseAttentionBackend.get_impl_cls / get_builder_cls / get_metadata_cls`: Wan picks
                      WanTransformerBlock_VSA from the env string (models/dits/wanvideo.py:628-629) and the denoising stage
                      builds VSA metadata only when the backend class IS VideoSparseAttentionBackend
                      (pipelines/stages/denoising.py:466), so the class identity is kept and the pipelines run unchanged.
  linear              @register_quantization_config("fvb200_bf16") Fvb200Bf16Config(QuantizationConfig) whose
                      get_quant_method returns Fvb200LinearMethod(LinearMethodBase)
                      (fastvideo/layers/quantization/__init__.py:13-45, base_config.py:17-140, layers/linear.py:80-156).
  linear (FP8)        @register_quantization_config("fvb200_fp8") Fvb200Fp8Config: Fvb200Fp8LinearMethod loads the same
                      bf16 weight, quantises it to e4m3 per output channel in process_weights_after_loading (the bf16
                      parameter is replaced, not kept) and applies ops.linear_fp8 (activations quantised per token).
  linear (INT8 w)     @register_quantization_config("fvb200_int8w") Fvb200Int8WeightConfig: Fvb200Int8WeightLinearMethod
                      loads the same bf16 weight, quantises it to int8 per output channel in process_weights_after_loading
                      (the bf16 parameter is replaced) and applies ops.linear_any (bf16 activations, fvb_linear_w8_sp).
  linear (W8A8)       @register_quantization_config("fvb200_w8a8") Fvb200W8A8Config: Fvb200W8A8LinearMethod loads and
                      quantises the weight like fvb200_int8w and applies ops.linear_any on an Int8Weight marked for int8
                      activations (quantised per token by fvb_quantize_int8_rows, then fvb_linear_w8a8_sp).
  custom ops          RMSNorm.forward_cuda (fastvideo/layers/layernorm.py:12-83) on fvb_rmsnorm_rope, and
                      CustomOp.dispatch_forward (fastvideo/layers/custom_op.py:53-57, hard-wired to forward_native) routed
                      to forward_cuda for the classes that got one.
  whole block         load_wan_block(): a reference WanTransformerBlock(_VSA)'s state_dict() -> wan_dit.WanBlock.

Training: the dense backend (through B200AttentionImpl, backward fvb_attention_bwd), the VSA impl (through
VideoSparseAttentionImpl: compact-layout backward on fvb_attention_sparse_bwd, fvb_vsa_combine_bwd_compact and
fvb_block_mean_bwd_compact; tile / untile as autograd permutations), RMSNorm.forward_cuda (backward fvb_rmsnorm_bwd) and
the fvb200_bf16 linear method (through linear_forward, backward fvb_linear_dgrad_bf16 / fvb_linear_wgrad_bf16 /
fvb_bias_grad_bf16) are differentiable when grad is enabled and an input requires grad; without grad they run the same
calls as before. The 8-bit backend and the FP8, INT8-weight and W8A8 linear methods are forward-only.

There is no CPU fallback anywhere: with non-CUDA tensors these classes raise FvbError exactly like the rest of the
package. uninstall() restores every patched attribute.
"""
from __future__ import annotations

import os
import types

import torch

from . import attention as _mirror
from . import ops
from ._lib import FvbError

DENSE_BACKEND_NAME = "FVB200_ATTN"
DENSE_8BIT_BACKEND_NAME = "FVB200_ATTN_8BIT"
QUANT_NAME = "fvb200_bf16"
QUANT_NAME_FP8 = "fvb200_fp8"
QUANT_NAME_INT8W = "fvb200_int8w"
QUANT_NAME_W8A8 = "fvb200_w8a8"

_state: types.SimpleNamespace | None = None


def available() -> bool:
    try:
        import fastvideo.attention.backends.abstract  # noqa: F401
        return True
    except Exception:  # noqa: BLE001 -- any import problem means "not inside a FastVideo checkout"
        return False


def _extend_enum(enum_cls, name: str):
    """Adds a member to an existing Enum class (what a maintainer does by editing platforms/interface.py:13-27)."""
    if name in enum_cls.__members__:
        return enum_cls[name]
    value = max(m.value for m in enum_cls) + 1
    member = object.__new__(enum_cls)
    member._name_ = name
    member._value_ = value
    member._sort_order_ = len(enum_cls._member_names_)
    enum_cls._member_names_.append(name)
    enum_cls._member_map_[name] = member
    enum_cls._value2member_map_[value] = member
    type.__setattr__(enum_cls, name, member)
    return member


def _define():
    """Creates the subclasses (needs `fastvideo` importable). Returns a namespace of classes."""
    from dataclasses import dataclass

    from fastvideo.attention.backends import abstract as A
    from fastvideo.attention.backends import video_sparse_attn as V
    from fastvideo.layers.linear import LinearBase, LinearMethodBase
    from fastvideo.layers.quantization.base_config import QuantizationConfig
    from fastvideo.models.utils import set_weight_attrs
    from torch.nn import Parameter

    ns = types.SimpleNamespace()

    # ------------------------------------------------------------------ dense attention
    @dataclass
    class Fvb200AttentionMetadata(A.AttentionMetadata):
        attn_mask: torch.Tensor | None = None

    class Fvb200AttentionMetadataBuilder(A.AttentionMetadataBuilder):
        def __init__(self) -> None:
            pass

        def prepare(self) -> None:
            pass

        def build(self, current_timestep: int = 0, attn_mask: torch.Tensor | None = None, **kwargs):
            return Fvb200AttentionMetadata(current_timestep=current_timestep, attn_mask=attn_mask)

    class Fvb200AttentionImpl(A.AttentionImpl):
        """SDPAImpl / FlashAttentionImpl contract (attention/backends/sdpa.py:106-147): [B, S, H, d] in and out."""

        def __init__(self, num_heads: int, head_size: int, softmax_scale: float | None = None, causal: bool = False,
                     num_kv_heads: int | None = None, prefix: str = "", **extra_impl_args) -> None:
            self._impl = _mirror.B200AttentionImpl(num_heads, head_size, causal=causal, softmax_scale=softmax_scale,
                                                   num_kv_heads=num_kv_heads, prefix=prefix)

        def forward(self, query, key, value, attn_metadata=None):
            return self._impl.forward(query, key, value, attn_metadata)

    class Fvb200AttentionBackend(A.AttentionBackend):
        accept_output_buffer: bool = True

        @staticmethod
        def get_supported_head_sizes() -> list[int]:
            return [128]

        @staticmethod
        def get_name() -> str:
            return DENSE_BACKEND_NAME

        @staticmethod
        def get_impl_cls():
            return Fvb200AttentionImpl

        @staticmethod
        def get_metadata_cls():
            return Fvb200AttentionMetadata

        @staticmethod
        def get_builder_cls():
            return Fvb200AttentionMetadataBuilder

    class Fvb200Attention8bitImpl(Fvb200AttentionImpl):
        """Fvb200AttentionImpl on the 8-bit attention (attention.B200Attention8bitImpl)."""

        def __init__(self, num_heads: int, head_size: int, softmax_scale: float | None = None, causal: bool = False,
                     num_kv_heads: int | None = None, prefix: str = "", **extra_impl_args) -> None:
            self._impl = _mirror.B200Attention8bitImpl(num_heads, head_size, causal=causal, softmax_scale=softmax_scale,
                                                       num_kv_heads=num_kv_heads, prefix=prefix)

    class Fvb200Attention8bitBackend(Fvb200AttentionBackend):
        @staticmethod
        def get_name() -> str:
            return DENSE_8BIT_BACKEND_NAME

        @staticmethod
        def get_impl_cls():
            return Fvb200Attention8bitImpl

    # ------------------------------------------------------------------ Video Sparse Attention
    @dataclass
    class Fvb200VideoSparseAttentionMetadata(V.VideoSparseAttentionMetadata):
        block_offsets: torch.Tensor | None = None  # int32 [n_tiles + 1]: first row of each tile, compact tile-major order
        row_block: torch.Tensor | None = None      # int32 [S]: compact row -> tile

    class Fvb200VideoSparseAttentionMetadataBuilder(V.VideoSparseAttentionMetadataBuilder):
        """Same build() signature and fields (video_sparse_attn.py:192-235); tables from fvb_vsa_tile_index."""

        def build(self, current_timestep, raw_latent_shape, patch_size, VSA_sparsity, device, cache_tile_buf=True,
                  **kwargs):
            m = _mirror.VideoSparseAttentionMetadataBuilder().build(current_timestep, raw_latent_shape, patch_size,
                                                                   VSA_sparsity, device, cache_tile_buf)
            return Fvb200VideoSparseAttentionMetadata(
                current_timestep=m.current_timestep, dit_seq_shape=tuple(m.dit_seq_shape), VSA_sparsity=m.VSA_sparsity,
                num_tiles=tuple(m.num_tiles), total_seq_length=m.total_seq_length,
                tile_partition_indices=m.tile_partition_indices,
                reverse_tile_partition_indices=m.reverse_tile_partition_indices,
                variable_block_sizes=m.variable_block_sizes, non_pad_index=m.non_pad_index,
                untile_combined_index=m.untile_combined_index, cache_tile_buf=cache_tile_buf,
                block_offsets=m.block_offsets, row_block=m.row_block)

    class Fvb200VideoSparseAttentionImpl(V.VideoSparseAttentionImpl):
        """preprocess_qkv -> forward(q, k, v, gate, md) -> postprocess_output, as DistributedAttention_VSA drives them
        (attention/layer.py:172-245). "Tiling" is a permutation into compact tile-major order (no zero rows).
        Differentiable (delegates to attention.VideoSparseAttentionImpl): with grad enabled and an input that requires
        grad, tiling and untiling are autograd permutations and forward runs the compact-layout VSA backward; the forward
        output is the same bits as without grad."""

        def __init__(self, num_heads: int, head_size: int, causal: bool = False, softmax_scale: float | None = None,
                     num_kv_heads: int | None = None, prefix: str = "", **extra_impl_args) -> None:
            self.prefix = prefix
            self._impl = _mirror.VideoSparseAttentionImpl(num_heads, head_size, causal=causal, softmax_scale=softmax_scale,
                                                          num_kv_heads=num_kv_heads, prefix=prefix)

        def tile(self, x, attn_metadata):
            return self._impl.tile(x, attn_metadata)

        def untile(self, x, attn_metadata):  # the reference passes the combined index; both forms are accepted
            if torch.is_tensor(attn_metadata):
                raise FvbError("Fvb200 VSA untile takes the metadata object (compact layout has no padded index)")
            return self._impl.untile(x, attn_metadata)

        def preprocess_qkv(self, qkv, attn_metadata):
            return self._impl.preprocess_qkv(qkv, attn_metadata)

        def postprocess_output(self, output, attn_metadata):
            return self._impl.postprocess_output(output, attn_metadata)

        def forward(self, query, key, value, gate_compress, attn_metadata):
            return self._impl.forward(query, key, value, gate_compress, attn_metadata)

    # ------------------------------------------------------------------ linear
    class Fvb200LinearMethod(LinearMethodBase):
        """UnquantizedLinearMethod's weight layout (layers/linear.py:120-156), applied by linear_forward (fvb_linear_bf16;
        differentiable when the input, the weight or the bias requires grad)."""

        def create_weights(self, layer, input_size_per_partition, output_partition_sizes, input_size, output_size,
                           params_dtype, **extra_weight_attrs) -> None:
            weight = Parameter(torch.empty(sum(output_partition_sizes), input_size_per_partition, dtype=params_dtype),
                               requires_grad=False)
            set_weight_attrs(weight, {"input_dim": 1, "output_dim": 0})
            layer.register_parameter("weight", weight)
            set_weight_attrs(weight, extra_weight_attrs)

        def apply(self, layer, x, bias=None):
            return linear_forward(x, layer.weight, bias)

    class Fvb200Bf16Config(QuantizationConfig):
        def get_name(self):
            return QUANT_NAME

        def get_supported_act_dtypes(self):
            return [torch.bfloat16]

        @classmethod
        def get_min_capability(cls) -> int:
            return 90

        @staticmethod
        def get_config_filenames() -> list[str]:
            return []

        @classmethod
        def from_config(cls, config):
            return cls()

        def get_quant_method(self, layer, prefix: str):
            return Fvb200LinearMethod() if isinstance(layer, LinearBase) else None

    class Fvb200Fp8LinearMethod(Fvb200LinearMethod):
        """Same bf16 weight parameter as Fvb200LinearMethod; after loading it becomes `weight` (float8_e4m3fn [N, K]) plus
        `weight_scale` (fp32 [N]), and apply() runs fvb_quantize_fp8_rows + fvb_linear_fp8."""

        def process_weights_after_loading(self, layer) -> None:
            w = layer.weight
            if not w.is_cuda:
                raise FvbError("fvb200_fp8 quantises its weights on the GPU: load the model onto a CUDA device")
            fw = ops.Fp8Weight.quantize(w.data.to(torch.bfloat16))
            layer.weight = Parameter(fw.q, requires_grad=False)  # drops the bf16 parameter
            layer.weight_scale = Parameter(fw.scale, requires_grad=False)

        def apply(self, layer, x, bias=None):
            if not x.is_cuda:
                raise FvbError("fvb200_fp8 linear needs CUDA tensors (there is no CPU fallback)")
            if layer.weight.dtype != torch.float8_e4m3fn:
                raise FvbError("fvb200_fp8 linear: weights are not quantised (process_weights_after_loading did not run)")
            if x.dtype != torch.bfloat16:
                raise FvbError(f"fvb200_fp8 linear takes bf16 activations (got {x.dtype})")
            w = ops.Fp8Weight(layer.weight, layer.weight_scale)
            b = None if bias is None else bias.to(torch.bfloat16)
            return ops.linear_fp8(x, w, b)

    class Fvb200Fp8Config(Fvb200Bf16Config):
        def get_name(self):
            return QUANT_NAME_FP8

        @classmethod
        def get_min_capability(cls) -> int:
            return 90  # e4m3 wgmma: sm_90a

        def get_quant_method(self, layer, prefix: str):
            return Fvb200Fp8LinearMethod() if isinstance(layer, LinearBase) else None

    class Fvb200Int8WeightLinearMethod(Fvb200LinearMethod):
        """Same bf16 weight parameter as Fvb200LinearMethod; after loading it becomes `weight` (int8 [N, K]) plus
        `weight_scale` (fp32 [N]), and apply() runs fvb_linear_w8_sp on the bf16 activations."""
        int8_activations = False  # Fvb200W8A8LinearMethod: quantise the activations too

        def process_weights_after_loading(self, layer) -> None:
            w = layer.weight
            if not w.is_cuda:
                raise FvbError("fvb200_int8w quantises its weights on the GPU: load the model onto a CUDA device")
            iw = ops.Int8Weight.quantize(w.data)
            layer.weight = Parameter(iw.q, requires_grad=False)  # drops the bf16 parameter
            layer.weight_scale = Parameter(iw.scale, requires_grad=False)

        def apply(self, layer, x, bias=None):
            if not x.is_cuda:
                raise FvbError("fvb200_int8w linear needs CUDA tensors (there is no CPU fallback)")
            if layer.weight.dtype != torch.int8:
                raise FvbError("fvb200_int8w linear: weights are not quantised (process_weights_after_loading did not run)")
            if x.dtype != torch.bfloat16:
                raise FvbError(f"fvb200_int8w linear takes bf16 activations (got {x.dtype})")
            w = ops.Int8Weight(layer.weight, layer.weight_scale, int8_activations=self.int8_activations)
            b = None if bias is None else bias.to(torch.bfloat16)
            return ops.linear_any(x, w, b)

    class Fvb200Int8WeightConfig(Fvb200Bf16Config):
        def get_name(self):
            return QUANT_NAME_INT8W

        @classmethod
        def get_min_capability(cls) -> int:
            return 90  # sm_90a wgmma GEMM

        def get_quant_method(self, layer, prefix: str):
            return Fvb200Int8WeightLinearMethod() if isinstance(layer, LinearBase) else None

    class Fvb200W8A8LinearMethod(Fvb200Int8WeightLinearMethod):
        """Fvb200Int8WeightLinearMethod whose apply() also quantises the bf16 activations to int8, one scale per token
        (fvb_quantize_int8_rows), and runs fvb_linear_w8a8_sp."""
        int8_activations = True

    class Fvb200W8A8Config(Fvb200Bf16Config):
        def get_name(self):
            return QUANT_NAME_W8A8

        @classmethod
        def get_min_capability(cls) -> int:
            return 90  # s8 wgmma: sm_90a

        def get_quant_method(self, layer, prefix: str):
            return Fvb200W8A8LinearMethod() if isinstance(layer, LinearBase) else None

    ns.__dict__.update(
        Fvb200AttentionMetadata=Fvb200AttentionMetadata, Fvb200AttentionMetadataBuilder=Fvb200AttentionMetadataBuilder,
        Fvb200AttentionImpl=Fvb200AttentionImpl, Fvb200AttentionBackend=Fvb200AttentionBackend,
        Fvb200Attention8bitImpl=Fvb200Attention8bitImpl, Fvb200Attention8bitBackend=Fvb200Attention8bitBackend,
        Fvb200VideoSparseAttentionMetadata=Fvb200VideoSparseAttentionMetadata,
        Fvb200VideoSparseAttentionMetadataBuilder=Fvb200VideoSparseAttentionMetadataBuilder,
        Fvb200VideoSparseAttentionImpl=Fvb200VideoSparseAttentionImpl, Fvb200LinearMethod=Fvb200LinearMethod,
        Fvb200Bf16Config=Fvb200Bf16Config, Fvb200Fp8LinearMethod=Fvb200Fp8LinearMethod, Fvb200Fp8Config=Fvb200Fp8Config,
        Fvb200Int8WeightLinearMethod=Fvb200Int8WeightLinearMethod, Fvb200Int8WeightConfig=Fvb200Int8WeightConfig,
        Fvb200W8A8LinearMethod=Fvb200W8A8LinearMethod, Fvb200W8A8Config=Fvb200W8A8Config)
    return ns


def linear_forward(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None) -> torch.Tensor:
    """Fvb200LinearMethod.apply (UnquantizedLinearMethod's F.linear, layers/linear.py:146-156): bf16(x w^T + bias) over the
    last axis of x on fvb_linear_bf16. With grad enabled and x, w or bias requiring grad it runs ops.LinearFn (the same
    forward call, backward on fvb_linear_dgrad_bf16 / fvb_linear_wgrad_bf16 / fvb_bias_grad_bf16); otherwise the plain call."""
    if not x.is_cuda:
        raise FvbError("fvb200_bf16 linear needs CUDA tensors (there is no CPU fallback)")
    if w.dtype != torch.bfloat16 or x.dtype != torch.bfloat16:
        raise FvbError(f"fvb200_bf16 linear is bf16 x bf16 (got x {x.dtype}, weight {w.dtype})")
    x2 = x.reshape(-1, x.shape[-1])
    if x2.stride(-1) != 1:
        x2 = x2.contiguous()
    b = None if bias is None else bias.to(torch.bfloat16)
    if torch.is_grad_enabled() and (x.requires_grad or w.requires_grad or (b is not None and b.requires_grad)):
        out = ops.LinearFn.apply(x2, w, b)
    else:
        out = ops.linear(x2, w, b)
    return out.reshape(*x.shape[:-1], w.shape[0])


def rms_norm_forward_cuda(self, x: torch.Tensor, residual: torch.Tensor | None = None):
    """RMSNorm.forward_cuda (the slot CustomOp leaves open, custom_op.py:36-37): x * rsqrt(mean(x^2) + eps) in fp32,
    cast to x.dtype, then * weight -- the product takes the promoted dtype when the weight is fp32 (layernorm.py:77-79)."""
    if residual is not None or self.variance_size_override is not None:
        return self.forward_native(x, residual)  # fused-add and partial-variance forms are not Wan hot-path inputs
    if not x.is_cuda or x.dtype != torch.bfloat16:
        raise FvbError("RMSNorm.forward_cuda (libfvb200) needs a CUDA bf16 tensor")
    D = x.shape[-1]
    if D != self.hidden_size:
        raise ValueError(f"Expected hidden_size to be {self.hidden_size}, but found: {D}")
    w = self.weight if self.has_weight else None
    w_bf16 = w is not None and w.dtype == torch.bfloat16
    if torch.is_grad_enabled() and (x.requires_grad or (w_bf16 and w.requires_grad)):
        out = _RmsNormFn.apply(x.reshape(-1, D), w if w_bf16 else None, self.variance_epsilon).view(x.shape)
        return out if w is None or w_bf16 else out * w
    out = x.reshape(-1, D).clone()
    if w_bf16:
        ops.rmsnorm_rope_(out, w.contiguous(), head_dim=128, eps=self.variance_epsilon)
        return out.view(x.shape)
    ones = torch.ones(D, dtype=torch.bfloat16, device=x.device)
    ops.rmsnorm_rope_(out, ones, head_dim=128, eps=self.variance_epsilon)
    out = out.view(x.shape)
    return out if w is None else out * w  # fp32 weight: promoted product, as in the reference


class _RmsNormFn(torch.autograd.Function):
    """bf16(bf16(x * rsqrt(mean(x^2) + eps)) * w) over rows of x [M, D], w bf16 [D] or None (ones): forward on
    fvb_rmsnorm_rope (the output of the no-grad call, bit for bit), backward on fvb_rmsnorm_bwd. An fp32 weight stays outside
    (the caller multiplies, and torch differentiates the product), so w here is only ever bf16."""

    @staticmethod
    def forward(ctx, x, w, eps):
        out = x.clone()
        ops.rmsnorm_rope_(out, w.contiguous() if w is not None else torch.ones(x.shape[1], dtype=torch.bfloat16, device=x.device),
                          head_dim=128, eps=eps)
        ctx.save_for_backward(x, w)
        ctx.eps = eps
        return out

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dy = dy.to(torch.bfloat16)
        if dy.stride(1) != 1 or dy.stride(0) % 8 != 0:
            dy = dy.contiguous()
        xc = x if x.stride(1) == 1 and x.stride(0) % 8 == 0 else x.contiguous()
        dx, dw = ops.rmsnorm_bwd(xc, w.contiguous() if w is not None else None, dy, ctx.eps, want_dw=ctx.needs_input_grad[1])
        return dx, dw, None


def _dispatch_forward(self):
    """CustomOp.dispatch_forward with the forward_cuda branch alive for ops that have one registered by install()."""
    from fastvideo.layers.custom_op import CustomOp
    own = type(self).__dict__.get("forward_cuda") or next(
        (c.__dict__["forward_cuda"] for c in type(self).__mro__ if "forward_cuda" in c.__dict__ and c is not CustomOp), None)
    if own is not None and getattr(own, "_fvb200", False) and torch.cuda.is_available():
        return self.forward_cuda
    return self.forward_native


def load_wan_block(block: torch.nn.Module, cfg=None):
    """Reference `WanTransformerBlock` / `WanTransformerBlock_VSA` module -> wan_dit.WanBlock (same parameter names)."""
    from . import wan_dit
    sd = block.state_dict()
    if cfg is None:
        D = sd["to_q.weight"].shape[0]
        cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=D // 128, ffn_dim=sd["ffn.fc_in.weight"].shape[0],
                                   num_layers=1, vsa="to_gate_compress.weight" in sd)
    return wan_dit.WanBlock(sd, "", cfg)


def device_supported() -> bool:
    """The library holds sm_90a code only, which runs on compute capability 9.0 (H100 / H800 / H200) and nowhere else."""
    return torch.cuda.is_available() and tuple(torch.cuda.get_device_capability()) == (9, 0)


def route_dense(selected: str | None, head_size: int, dtype, force: bool = False) -> str | None:
    """Which dense backend of this package serves a request for the AttentionBackendEnum member named `selected` (None: no
    preference): the qualified class name, or None to leave the request to the platform. bf16, head_size 128 and a
    compute capability 9.0 device (or `force`) are required. FVB200_ATTN_8BIT is served only when selected by name; the
    bf16 backend also takes FLASH_ATTN / TORCH_SDPA / no-preference requests unless FVB200_ATTENTION=0."""
    ok = (force or device_supported()) and head_size == 128 and dtype == torch.bfloat16
    if selected == DENSE_8BIT_BACKEND_NAME:
        if not ok:
            raise ValueError(f"{DENSE_8BIT_BACKEND_NAME} supports bf16 with head_size 128 on sm_90 only")
        return f"{__name__}.Fvb200Attention8bitBackend"
    if (ok and selected in (None, "FLASH_ATTN", "TORCH_SDPA", DENSE_BACKEND_NAME)
            and os.environ.get("FVB200_ATTENTION", "1") != "0"):
        return f"{__name__}.Fvb200AttentionBackend"
    if selected == DENSE_BACKEND_NAME:
        raise ValueError(f"{DENSE_BACKEND_NAME} supports bf16 with head_size 128 on sm_90 only")
    return None


def install(dense: bool = True, vsa_backend: bool = True, linear: bool = True, custom_ops: bool = True,
            force: bool | None = None):
    """Registers everything (idempotent). `force=True` routes the dense backend even when the current device is not
    sm_90 (used by the CPU registration test); by default it follows FVB200_FORCE=1 or device_supported()."""
    global _state
    if _state is not None:
        return _state.ns
    if not available():
        raise FvbError("fastvideo is not importable: fastvideo_b200.plugin.install() registers INTO a FastVideo checkout")
    import sys

    from fastvideo.attention.backends import video_sparse_attn as V
    from fastvideo.platforms import current_platform
    from fastvideo.platforms.interface import AttentionBackendEnum

    ns = _define()
    mod = sys.modules[__name__]
    for k, v in ns.__dict__.items():  # resolve_obj_by_qualname("fastvideo_b200.plugin.<Class>") must find them
        v.__module__ = __name__
        v.__qualname__ = k
        setattr(mod, k, v)
    undo = []

    def patch(obj, name, value):
        had = name in obj.__dict__
        undo.append((obj, name, obj.__dict__.get(name), had))
        setattr(obj, name, value)

    if force is None:
        force = os.environ.get("FVB200_FORCE", "0") == "1"

    if dense:
        _extend_enum(AttentionBackendEnum, DENSE_BACKEND_NAME)
        _extend_enum(AttentionBackendEnum, DENSE_8BIT_BACKEND_NAME)
        plat_cls = type(current_platform) if not isinstance(current_platform, type) else current_platform
        orig = plat_cls.__dict__.get("get_attn_backend_cls") or getattr(plat_cls, "get_attn_backend_cls")
        orig_fn = orig.__func__ if isinstance(orig, classmethod) else orig

        def get_attn_backend_cls(cls, selected_backend, head_size, dtype):
            name = None if selected_backend is None else selected_backend.name
            routed = route_dense(name, head_size, dtype, force)
            return routed if routed is not None else orig_fn(cls, selected_backend, head_size, dtype)

        patch(plat_cls, "get_attn_backend_cls", classmethod(get_attn_backend_cls))
        try:  # the resolution is functools-cached on its arguments (attention/selector.py:239)
            from fastvideo.attention import selector
            selector._cached_get_attn_backend.cache_clear()
        except Exception:  # noqa: BLE001
            pass

    if vsa_backend:
        B = V.VideoSparseAttentionBackend
        patch(B, "get_impl_cls", staticmethod(lambda: ns.Fvb200VideoSparseAttentionImpl))
        patch(B, "get_builder_cls", staticmethod(lambda: ns.Fvb200VideoSparseAttentionMetadataBuilder))
        patch(B, "get_metadata_cls", staticmethod(lambda: ns.Fvb200VideoSparseAttentionMetadata))
        patch(B, "get_supported_head_sizes", staticmethod(lambda: [128]))

    if linear:
        from fastvideo.layers import quantization as Q
        if QUANT_NAME not in Q.QUANTIZATION_METHODS:
            Q.register_quantization_config(QUANT_NAME)(ns.Fvb200Bf16Config)
        if QUANT_NAME_FP8 not in Q.QUANTIZATION_METHODS:
            Q.register_quantization_config(QUANT_NAME_FP8)(ns.Fvb200Fp8Config)
        if QUANT_NAME_INT8W not in Q.QUANTIZATION_METHODS:
            Q.register_quantization_config(QUANT_NAME_INT8W)(ns.Fvb200Int8WeightConfig)
        if QUANT_NAME_W8A8 not in Q.QUANTIZATION_METHODS:
            Q.register_quantization_config(QUANT_NAME_W8A8)(ns.Fvb200W8A8Config)

    if custom_ops:
        from fastvideo.layers.custom_op import CustomOp
        from fastvideo.layers.layernorm import RMSNorm
        rms_norm_forward_cuda._fvb200 = True
        patch(RMSNorm, "forward_cuda", rms_norm_forward_cuda)
        patch(CustomOp, "dispatch_forward", _dispatch_forward)

    _state = types.SimpleNamespace(ns=ns, undo=undo)
    return ns


def uninstall() -> None:
    global _state
    if _state is None:
        return
    for obj, name, old, had in reversed(_state.undo):
        if had:
            setattr(obj, name, old)
        else:
            delattr(obj, name)
    try:
        from fastvideo.attention import selector
        selector._cached_get_attn_backend.cache_clear()
    except Exception:  # noqa: BLE001
        pass
    _state = None


__all__ = ["available", "install", "uninstall", "load_wan_block", "linear_forward", "rms_norm_forward_cuda", "route_dense", "DENSE_BACKEND_NAME",
           "DENSE_8BIT_BACKEND_NAME", "QUANT_NAME", "QUANT_NAME_FP8",
           "QUANT_NAME_INT8W"]
