"""CPU: the 8-bit attention restatement (tests/attn8_ref.py) -- its error against exact attention and why Q K^T is INT8,
the vt8 key-slot order, which attention of the Wan block it replaces -- and the plug-in's routing of FVB200_ATTN_8BIT."""
import pytest
import torch

import attn8_ref
import fp8_ref


def _qkv(g, Sq, Skv, q_gain=2.0):
    """Random q, k, v with a per-channel bias on K (what the K smoothing removes)."""
    q = (torch.randn(1, Sq, 1, 128, generator=g) * q_gain).bfloat16()
    k = (torch.randn(1, Skv, 1, 128, generator=g) + 3 * torch.randn(128, generator=g)).bfloat16()
    v = torch.randn(1, Skv, 1, 128, generator=g).bfloat16()
    return q, k, v


def test_restatement_error_against_exact_attention_and_the_e4m3_qk_alternative():
    """INT8 Q K^T with per-token scales and a smoothed K: 3.5-3.8 % rel-L2 from fp64 attention here (1024 keys); the same
    with e4m3 Q and K (per-token scale, no smoothing): 10-21 %. bf16 rounding of the output alone: 0.17 %."""
    g = torch.Generator().manual_seed(0)
    for q_gain in (1.0, 3.0):
        q, k, v = _qkv(g, 128, 1024, q_gain)
        qz = attn8_ref.quantize(q, k, v)
        exact = attn8_ref.exact_attention(q, k, v)
        e_int8 = attn8_ref.rel_l2(attn8_ref.attention(qz, 128 ** -0.5), exact)
        q8e, sqe = fp8_ref.quantize_fp8_rows(q.float().transpose(1, 2))
        k8e, ske = fp8_ref.quantize_fp8_rows(k.float().transpose(1, 2))
        qe = dict(qz, q8=q8e.float(), q_scale=sqe, k8=k8e.float(), k_scale=ske)
        e_e4m3 = attn8_ref.rel_l2(attn8_ref.attention(qe, 128 ** -0.5), exact)
        assert 0.01 < e_int8 < 0.05, e_int8
        assert e_e4m3 > 2.5 * e_int8, (e_e4m3, e_int8)


def test_the_e4m3_p_is_part_of_the_error():
    g = torch.Generator().manual_seed(1)
    q, k, v = _qkv(g, 64, 512)
    qz = attn8_ref.quantize(q, k, v)
    a = attn8_ref.attention(qz, 128 ** -0.5)
    b = attn8_ref.attention(qz, 128 ** -0.5, p_e4m3=False)
    assert 1e-3 < attn8_ref.rel_l2(a, b) < 5e-2


def test_vt8_slot_order():
    # the accumulator columns 2t, 2t+1, 8+2t, 9+2t of a 16-key group are A-fragment slots 4t .. 4t+3
    assert attn8_ref.PERM16 == [0, 1, 8, 9, 2, 3, 10, 11, 4, 5, 12, 13, 6, 7, 14, 15]
    g = torch.Generator().manual_seed(2)
    q, k, v = _qkv(g, 8, 100)
    off = torch.tensor([0, 40, 100], dtype=torch.int32)
    qz = attn8_ref.quantize(q, k, v, kv_off=off)
    assert qz["blocks"] == [(0, 40), (40, 60)]
    v8 = qz["v8"].view(torch.uint8)
    for blk, (row0, vlen) in enumerate(qz["blocks"]):
        for j in range(64):
            key = attn8_ref.SLOT_KEY[j]
            want = v8[0, 0, row0 + key] if key < vlen else torch.zeros(128, dtype=torch.uint8)
            assert torch.equal(qz["vt8"][0, 0, blk, :, j], want), (blk, j)


def test_int8_rows_zero_and_rounding():
    x = torch.zeros(3, 128)
    x[1, :5] = torch.tensor([127.0, 0.5, -1.5, 2.5, 3.25])  # amax 127: inv = 1, ties go to even
    x[2] = 5.0
    q, s = attn8_ref.quantize_rows_int8(x)
    assert s[0] == 1.0 and (q[0] == 0).all()
    assert q[1, :5].tolist() == [127, 0, -2, 2, 3] and s[1] == 1.0
    assert (q[2] == 127).all()


def test_oracle_routing_sends_exactly_the_self_attention_to_the_restatement(monkeypatch):
    from oracle import wan_ref
    from oracle.gen_golden import _rand_block_sd
    g = torch.Generator().manual_seed(3)
    D, H, L, S, seq = 256, 2, 8, 8, (1, 2, 4)
    sd = _rand_block_sd(D, 512, H, False, g)
    x = torch.randn(1, S, D, generator=g).bfloat16()
    ctx = torch.randn(1, L, D, generator=g).bfloat16()
    temb6 = (torch.randn(1, 6, D, generator=g) * 0.5).bfloat16()
    cos, sin = wan_ref.rotary_tables(seq, [44, 42, 42])
    routed, plain = [], []
    real8, real_sdpa = attn8_ref.attention_8bit_bshd, wan_ref.sdpa
    monkeypatch.setattr(attn8_ref, "attention_8bit_bshd", lambda q, k, v: (routed.append(k.shape), real8(q, k, v))[1])
    monkeypatch.setattr(wan_ref, "sdpa", lambda q, k, v, *a, **kw: (plain.append(k.shape), real_sdpa(q, k, v, *a, **kw))[1])
    block, vsa = wan_ref.wan_block, wan_ref.video_sparse_attn
    with torch.no_grad():
        y8 = attn8_ref.wan_block_attn8(x, ctx, temb6, sd, "", H, cos, sin)
    assert wan_ref.wan_block is block and wan_ref.video_sparse_attn is vsa
    assert routed == [(1, S, H, D // H)]  # the self-attention: keys are the block's own tokens
    assert plain == [(1, L, H, D // H)]   # the cross-attention: keys are the text states
    with torch.no_grad():
        y16 = wan_ref.wan_block(x, ctx, temb6, sd, "", H, cos, sin)
    rel = attn8_ref.rel_l2(y8.float(), y16.float())
    assert 1e-4 < rel < 1e-1, rel


def test_plugin_routes_fvb200_attn_8bit_only_on_a_9_0_device(monkeypatch):
    from fastvideo_b200 import plugin
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    name = plugin.DENSE_8BIT_BACKEND_NAME
    assert name == "FVB200_ATTN_8BIT"
    for cap in ((10, 0), (8, 0), (9, 1)):
        monkeypatch.setattr(torch.cuda, "get_device_capability", lambda *a, cap=cap: cap)
        with pytest.raises(ValueError):
            plugin.route_dense(name, 128, torch.bfloat16)
    monkeypatch.setattr(torch.cuda, "get_device_capability", lambda *a: (9, 0))
    assert plugin.route_dense(name, 128, torch.bfloat16) == "fastvideo_b200.plugin.Fvb200Attention8bitBackend"
    for hs, dt in ((64, torch.bfloat16), (128, torch.float16)):
        with pytest.raises(ValueError):
            plugin.route_dense(name, hs, dt)
    # it is never chosen for the bf16 names or "no preference"
    for sel in (None, "FLASH_ATTN", "TORCH_SDPA", plugin.DENSE_BACKEND_NAME):
        assert plugin.route_dense(sel, 128, torch.bfloat16) == "fastvideo_b200.plugin.Fvb200AttentionBackend"
    assert plugin.route_dense("SAGE_ATTN", 128, torch.bfloat16) is None
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(ValueError):
        plugin.route_dense(name, 128, torch.bfloat16)
