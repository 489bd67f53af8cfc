"""CPU: the compact-layout VSA grad path (VideoSparseAttentionImpl.forward with an input that requires grad) refuses the
pair-union sparse kernel, as the padded layout does, instead of running another kernel than the no-grad call would."""
from types import SimpleNamespace

import pytest
import torch


def test_compact_grad_path_refuses_the_pair_union_kernel(monkeypatch):
    from fastvideo_b200 import ops, vsa
    from fastvideo_b200.attention import VideoSparseAttentionImpl
    monkeypatch.setattr(vsa, "SPARSE_KERNEL", "union")
    q = torch.zeros(1, 64, 1, 128, dtype=torch.bfloat16, requires_grad=True)
    vbs = torch.tensor([64], dtype=torch.int32)
    md = SimpleNamespace(VSA_sparsity=0.0, variable_block_sizes=vbs, block_offsets=torch.tensor([0, 64], dtype=torch.int32),
                         row_block=torch.zeros(64, dtype=torch.int32))
    with pytest.raises(ops.FvbError):
        VideoSparseAttentionImpl(num_heads=1, head_size=128).forward(q, q, q, q, md)
