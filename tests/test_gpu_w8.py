"""GPU: INT8 weight-only linears (bf16 activations) -- fvb_linear_w8_sp against an fp64 evaluation of its formula, its
sequence-parallel options, and every Wan path with WanDiTConfig.int8_weights against the oracle with exactly the engine's
INT8 weights routed to the restatement (tests/w8_ref.py). int8 -> bf16 is exact, so the arithmetic is the bf16 engine's
apart from accumulation order, and every model case is held to the bf16 parity gate against the routed oracle."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import attn8_ref
import w8_ref
from conftest import ROOT
from oracle import causal_ref, vsa_index, wan_ref
from util import assert_bf16_parity, rel_l2

pytestmark = pytest.mark.gpu


def cuda_sd(sd):
    return {k: v.cuda() for k, v in sd.items()}


# ------------------------------------------------------------------------------------------------ fvb_linear_w8_sp
def ref_linear_w8(x, wq, ws, b, epi, resid, gate, gate_rows):
    """(fp64 value of the formula, the formula with its fp32 / bf16 rounding points) for fvb_linear_w8_sp. bf16 x int8
    products are exact in fp64 and so are their sums here, so the fp64 GEMM (on the GPU for speed) is the exact accumulator."""
    acc = x.double() @ wq.double().t()
    exact = acc * ws.double()[None, :]
    y32 = acc.float() * ws[None, :]
    if b is not None:
        exact = exact + b.double()
        y32 = y32 + b.float()
    y = y32.bfloat16().float()
    if gate is not None:
        g = gate if gate_rows == 0 else gate.repeat_interleave(gate_rows, 0)[: x.shape[0]]
    if epi == 0: return exact, y.bfloat16()
    if epi == 1: return F.gelu(exact, approximate="tanh"), F.gelu(y, approximate="tanh").bfloat16()
    if epi == 2: return resid.double() + exact * g.double(), resid.float() + y * g
    if epi == 3: return resid.double() + exact * g.double(), (resid.float() + y * g).bfloat16()
    if epi == 7: return resid.double() + exact * g.double(), (resid.float() + (y * g).bfloat16().float()).bfloat16()
    if epi == 4: return resid.double() + exact, (resid.float() + y).bfloat16()


# (M, N, K, epilogue, gate_rows): small M, M = 4680, K = 5120 / 13 824, N multiples of 8 and of 128, every epilogue
CASES = [(1, 1536, 256, 0, 0), (333, 200, 200, 0, 0), (300, 64, 512, 0, 0), (1000, 1536, 1536, 1, 0), (1000, 1536, 1536, 2, 0),
         (777, 1536, 1536, 3, 0), (777, 1536, 1536, 3, 100), (777, 1536, 1536, 7, 128), (777, 1536, 1536, 4, 0),
         (4680, 5120, 5120, 0, 0), (4680, 5120, 5120, 7, 1560), (2048, 5120, 13824, 4, 0), (512, 13824, 5120, 1, 0),
         (4680, 1000, 5120, 2, 0)]


def _case(M, N, K, epi, gate_rows):
    from fastvideo_b200 import ops
    torch.manual_seed(M + N + K + epi)
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda").bfloat16()
    resid = torch.randn(M, N, device="cuda").bfloat16() if epi >= 2 else None
    gate = None
    if epi in (2, 3, 7):
        gate = torch.randn(N, device="cuda") if gate_rows == 0 else torch.randn((M + gate_rows - 1) // gate_rows, N, device="cuda")
    return x, ops.Int8Weight.quantize(w), b, resid, gate


@pytest.mark.parametrize("M,N,K,epi,gate_rows", CASES)
def test_linear_w8_matches_formula(M, N, K, epi, gate_rows):
    """bf16 parity against the fp64 value of the formula in include/fvb200.h, and fewer than 2 % of the bf16 outputs off
    the formula's own rounding (the bf16 linear tests' rule: only the fp32 accumulation order differs)."""
    from fastvideo_b200 import ops
    x, w, b, resid, gate = _case(M, N, K, epi, gate_rows)
    out = ops.linear_any(x, w, b, epi, resid, gate, gate_rows=gate_rows)
    exact, rounded = ref_linear_w8(x, w.q, w.scale, b, epi, resid, gate, gate_rows)
    if epi == 2:  # fp32 output
        assert out.dtype == torch.float32
        assert rel_l2(out, rounded) < 1e-4
        return
    assert_bf16_parity(out, exact, rounded, name=f"linear_w8 epi{epi}")
    mism = (out.float() != rounded.float()).float().mean().item()
    print(f"linear_w8 {M}x{N}x{K} epi{epi} gate_rows {gate_rows}: {mism:.4f} of outputs off the formula's rounding")
    assert mism < 0.02


def test_linear_w8_sp_options_bit_equal_to_plain_call():
    """x_seg_len / x_seg_stride (the all-to-all receive buffer read as [token, all heads * d]) and out_col_offsets (heads
    scattered into a send buffer) give exactly the plain call's outputs, rearranged."""
    from fastvideo_b200 import ops
    torch.manual_seed(7)
    M, K, N, seg = 300, 1024, 768, 256
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = ops.Int8Weight.quantize((torch.randn(N, K, device="cuda") / 32).bfloat16())
    b = torch.randn(N, device="cuda").bfloat16()
    plain = ops.linear_any(x, w, b)
    # A segmented: K split into 4 segments of 256 that live [src][token][seg] apart
    buf = x.view(M, K // seg, seg).permute(1, 0, 2).contiguous()  # [4, M, 256]
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.linear_sp(buf, M, K, seg, w, b, out, N, x_seg_len=seg, x_seg_stride=M * seg)
    assert torch.equal(out, plain)
    # column blocks of 128 scattered: block j goes to dest (j % 2), slot j // 2 of a [2, M, 3, 128] buffer
    send = torch.zeros(2, M, N // 256, 128, device="cuda", dtype=torch.bfloat16)
    offs = torch.tensor([(j % 2) * M * (N // 2) + (j // 2) * 128 for j in range(N // 128)], device="cuda", dtype=torch.int64)
    ops.linear_sp(x, M, K, K, w, b, send, N // 2, out_col_offsets=offs)
    back = send.permute(1, 2, 0, 3).reshape(M, N)  # [token, slot, dest, d] -> columns in j order
    assert torch.equal(back, plain)
    # and a residual epilogue through the same entry point
    r = torch.randn(M, N, device="cuda").bfloat16()
    assert torch.equal(ops.linear_any(x, w, b, ops.EPI_RESID_BF16, resid=r), (r.float() + plain.float()).bfloat16())


def test_linear_w8_rejects_bad_arguments():
    from fastvideo_b200 import ops
    x, w, b, _, _ = _case(64, 128, 256, 0, 0)
    with pytest.raises(ops.FvbError):
        ops.linear_any(x[:, :128], w)  # K mismatch
    out = torch.empty(64, 128, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ops.FvbError):  # column-block offsets need N % 128 == 0
        ops.linear_sp(x, 64, 256, 256, w[:64], None, out, 128, out_col_offsets=torch.zeros(1, device="cuda", dtype=torch.int64))


# ------------------------------------------------------------------------------------------------ Wan block / model
def _rope(seq, d):
    return wan_ref.rotary_tables(seq, [d - 4 * (d // 6), 2 * (d // 6), 2 * (d // 6)])


def _f32(sd):
    return {k: v.float() for k, v in sd.items()}


def _attn32(q, k, v):
    return wan_ref.attention_fp32(q, k, v)[0]


def _block_cfg(g, **kw):
    from fastvideo_b200 import wan_dit
    D, H = g["x"].shape[-1], g["heads"]
    return wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=H, ffn_dim=g["sd"]["ffn.fc_in.weight"].shape[0],
                                num_layers=1, **kw)


@pytest.mark.parametrize("name", ["wan_block_dense", "wan_block_i2v"])
def test_block_w8_against_routed_oracle(golden_dir, name):
    from fastvideo_b200 import ops, wan_dit
    g = torch.load(os.path.join(golden_dir, name + ".pt"))
    D, H = g["x"].shape[-1], g["heads"]
    outs = {}
    for int8 in (True, False):
        cfg = _block_cfg(g, int8_weights=int8)
        blk = wan_dit.WanBlock(cuda_sd(g["sd"]), "", cfg)
        if int8:
            for n in wan_dit.INT8_LINEARS:
                assert getattr(blk, n) is None or isinstance(getattr(blk, n), ops.Int8Weight), n
        lay = wan_dit.make_layout(g["seq"], cfg, "cuda")
        outs[int8] = wan_dit.block_forward(g["x"][0].cuda(), blk, g["ctx"][0].cuda(), g["temb6"].cuda(), lay, cfg)
    cos, sin = _rope(g["seq"], D // H)
    with torch.no_grad():
        yb = w8_ref.wan_block_w8(g["x"], g["ctx"], g["temb6"], g["sd"], "", H, cos, sin)
        y32 = w8_ref.wan_block_w8(g["x"].float(), g["ctx"].float(), g["temb6"].float(), _f32(g["sd"]), "", H, cos, sin,
                                  attn_fn=_attn32)
    e, floor = assert_bf16_parity(outs[True], y32[0], yb[0], name=f"int8w {name}")
    print(f"int8w {name}: relL2 {e:.3e} vs routed fp32 oracle (bf16 floor {floor:.3e}); {rel_l2(outs[True], outs[False]):.3e} "
          f"from the bf16 engine; {rel_l2(outs[True], g['y_fp32'][0]):.3e} from the fp32 oracle")
    assert rel_l2(outs[True], outs[False]) < 2e-2  # CPU measurement: the INT8-weight oracle is 7-8e-3 from the bf16 one


def _model(golden_dir, **kw):
    from fastvideo_b200 import wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_model_dense.pt"))
    sd = cuda_sd(g["sd"])
    cfg = wan_dit.WanDiTConfig(hidden_size=sd["proj_out.weight"].shape[1], num_attention_heads=g["heads"],
                               ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0], num_layers=2,
                               text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1], **kw)
    return g, cfg, wan_dit.WanDiT(cfg, sd)


def test_model_w8_against_routed_oracle(golden_dir):
    from fastvideo_b200 import ops, wan_dit
    g, cfg, model = _model(golden_dir, int8_weights=True)
    args = (g["latents"].cuda(), g["text"].cuda(), g["timestep"].cuda())
    y = model.forward(*args)
    y_bf16 = _model(golden_dir)[2].forward(*args)
    with torch.no_grad():
        yb = w8_ref.wan_model_w8(g["latents"], g["text"], g["timestep"], g["sd"], g["heads"])
        y32 = w8_ref.wan_model_w8(g["latents"].float(), g["text"].float(), g["timestep"], _f32(g["sd"]), g["heads"],
                                  attn_fn=_attn32)
    e, floor = assert_bf16_parity(y, y32, yb, name="int8w model")
    print(f"int8w model: relL2 {e:.3e} vs routed fp32 oracle (bf16 floor {floor:.3e}); {rel_l2(y, y_bf16):.3e} from the bf16 "
          f"engine")
    assert rel_l2(y, y_bf16) < 2e-2
    for blk in model.blocks:  # no bf16 copy of a quantised weight is left on the block
        for n in wan_dit.INT8_LINEARS:
            assert getattr(blk, n) is None or isinstance(getattr(blk, n), ops.Int8Weight)
        assert not [k for k, v in vars(blk).items() if torch.is_tensor(v) and v.dim() == 2 and v.dtype == torch.bfloat16]


def test_block_vsa_w8_against_routed_oracle():
    """The VSA block of test_gpu_fp8 with INT8 weights (including the gate rows of w_qkv): the row criteria of
    test_gpu_wan.test_block_vsa_against_oracle (median row relL2 < 1e-2) against the routed oracle."""
    from fastvideo_b200 import wan_dit
    from oracle.gen_golden import _rand_block_sd
    g = torch.Generator().manual_seed(5)
    D, H, F_, L = 256, 2, 512, 24
    seq = (5, 6, 7)
    S = int(np.prod(seq))
    sd = _rand_block_sd(D, F_, H, True, g)
    x = torch.randn(1, S, D, generator=g).bfloat16()
    ctx = torch.randn(1, L, D, generator=g).bfloat16()
    temb6 = (torch.randn(1, 6, D, generator=g) * 0.5).bfloat16()
    cos, sin = wan_ref.rotary_tables(seq, [44, 42, 42])
    tile = (4, 4, 4)
    vbs = torch.from_numpy(vsa_index.variable_block_sizes(seq, tile))
    meta = dict(tile_partition=torch.from_numpy(vsa_index.tile_partition_indices(seq, tile)),
                untile_combined=torch.from_numpy(vsa_index.untile_combined_index(seq, tile)),
                non_pad=torch.from_numpy(vsa_index.non_pad_index(vbs.numpy(), 64)), vbs=vbs, s_pad=vbs.numel() * 64,
                topk=vsa_index.compute_topk(0.5, vbs.numel()))
    with torch.no_grad():
        y_ref = w8_ref.wan_block_w8(x, ctx, temb6, sd, "", H, cos, sin, vsa_meta=meta)
    outs = {}
    for int8 in (True, False):
        cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=H, ffn_dim=F_, num_layers=1, vsa=True, int8_weights=int8)
        blk = wan_dit.WanBlock(cuda_sd(sd), "", cfg)
        lay = wan_dit.make_layout(seq, cfg, "cuda", vsa_sparsity=0.5)
        outs[int8] = wan_dit.block_forward(x[0].cuda()[lay.perm], blk, ctx[0].cuda(), temb6.cuda(), lay, cfg)[lay.inv_perm]
    y = outs[True]
    err_rows = (y.float().cpu() - y_ref[0].float()).norm(dim=-1) / y_ref[0].float().norm(dim=-1)
    print(f"int8w VSA block: median row relL2 {err_rows.median().item():.3e} vs routed oracle, "
          f"{rel_l2(y, outs[False]):.3e} from the bf16 engine")
    assert err_rows.median().item() < 1e-2
    assert (err_rows < 3e-2).float().mean().item() > 0.9


def test_block_w8_with_attention_8bit(golden_dir):
    """int8_weights + attention_8bit on the dense block, against the oracle with its self-attention on the 8-bit restatement
    and its linears on INT8 weights: the 1e-2 bound of test_gpu_attention_8bit for that path."""
    from fastvideo_b200 import wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_block_dense.pt"))
    D, H = g["x"].shape[-1], g["heads"]
    cfg = _block_cfg(g, int8_weights=True, attention_8bit=True)
    blk = wan_dit.WanBlock(cuda_sd(g["sd"]), "", cfg)
    lay = wan_dit.make_layout(g["seq"], cfg, "cuda")
    y = wan_dit.block_forward(g["x"][0].cuda(), blk, g["ctx"][0].cuda(), g["temb6"].cuda(), lay, cfg)
    cos, sin = _rope(g["seq"], D // H)
    with torch.no_grad(), w8_ref._wan_block_linears_in_int8(g["sd"], [""]):
        y_ref = attn8_ref.wan_block_attn8(g["x"], g["ctx"], g["temb6"], g["sd"], "", H, cos, sin)
    e = rel_l2(y, y_ref[0])
    print(f"int8w + attention_8bit block: relL2 {e:.3e} vs routed oracle")
    assert e <= 1e-2


# ------------------------------------------------------------------------------------------------ causal rollout
def test_causal_block_rollout_w8_against_routed_oracle(golden_dir):
    """The golden causal block rollout (sink frame, eviction, ring wrap) with INT8 weights, call by call."""
    from fastvideo_b200 import causal_wan, wan_dit
    from fastvideo_b200.rope import get_rotary_pos_embed
    g = torch.load(os.path.join(golden_dir, "wan_causal_block.pt"))
    D, H = g["sd"]["to_q.weight"].shape[0], g["heads"]
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=H, ffn_dim=g["sd"]["ffn.fc_in.weight"].shape[0],
                               num_layers=1, int8_weights=True)
    grid, nf = tuple(g["grid"]), g["frames_per_call"]
    fs = grid[0] * grid[1]
    W, S = g["window_frames"], g["sink_frames"]
    ccfg = causal_wan.CausalConfig(local_attn_size=W, sink_size=S, num_frames_per_block=nf)
    blk = wan_dit.WanBlock(cuda_sd(g["sd"]), "", cfg)
    cache = causal_wan.KVCache(W * fs, H, cfg.head_dim, "cuda", S * fs)
    xc = causal_wan.CrossAttnCache()
    ctx = g["ctx"][0].cuda()
    rb, r32 = causal_ref.new_kv_cache(1, W * fs, H, 128), causal_ref.new_kv_cache(1, W * fs, H, 128, torch.float32)
    xb, x32 = {"is_init": False}, {"is_init": False}
    sd32 = _f32(g["sd"])
    for i, c in enumerate(g["calls"]):
        cos, sin = get_rotary_pos_embed((nf, ) + grid, [44, 42, 42], start_frame=c["start_frame"], keep_f64=True)
        cs = c["start_frame"] * fs
        y = causal_wan.causal_block_forward(c["x"][0].cuda(), blk, ctx, c["temb"][0].cuda(), cos.cuda(), sin.cuda(), cache, xc,
                                            cs, cfg, ccfg, frame_seqlen=fs)
        with torch.no_grad():
            yb = w8_ref.causal_block_w8(c["x"], g["ctx"], c["temb"], g["sd"], "", H, cos, sin, rb, cs, W, S, fs, crossattn_cache=xb)
            y32 = w8_ref.causal_block_w8(c["x"].float(), g["ctx"].float(), c["temb"].float(), sd32, "", H, cos, sin, r32, cs, W, S,
                                         fs, crossattn_cache=x32)
        e, floor = assert_bf16_parity(y, y32[0], yb[0], name=f"int8w causal block call {i}")
        print(f"int8w causal block call {i}: relL2 {e:.3e} (floor {floor:.3e}); {rel_l2(y, c['y_ref_bf16'][0]):.3e} from the "
              f"bf16 reference")
        assert cache.local_end_index == c["local_end_index"]
    assert cache.head != 0


def _causal_model(golden_dir, int8):
    from fastvideo_b200 import causal_wan, wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_causal_model.pt"))
    sd = cuda_sd(g["sd"])
    cfg = wan_dit.WanDiTConfig(hidden_size=sd["proj_out.weight"].shape[1], num_attention_heads=g["heads"],
                               ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0], num_layers=2,
                               text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1], text_len=g["text_len"],
                               int8_weights=int8)
    ccfg = causal_wan.CausalConfig(local_attn_size=g["window_frames"], sink_size=g["sink_frames"],
                                   num_frames_per_block=g["frames_per_call"])
    return g, cfg, causal_wan.CausalWanDiT(cfg, sd, ccfg)


def test_causal_model_rollout_w8_against_routed_oracle(golden_dir):
    g, cfg, model = _causal_model(golden_dir, True)
    H, W, S = g["heads"], g["window_frames"], g["sink_frames"]
    c0 = g["calls"][0]["latents"]
    fs = (c0.shape[3] // 2) * (c0.shape[4] // 2)
    kv, xc = model.new_caches(fs, "cuda")
    text = g["text"].cuda()
    mk = lambda dt: [causal_ref.new_kv_cache(1, W * fs, H, 128, dt) for _ in range(2)]
    kb, k32 = mk(torch.bfloat16), mk(torch.float32)
    xb, x32 = [{"is_init": False} for _ in range(2)], [{"is_init": False} for _ in range(2)]
    sd32 = _f32(g["sd"])
    for i, c in enumerate(g["calls"]):
        y = model.forward_inference(c["latents"].cuda(), text, c["timestep"].cuda(), kv, xc, current_start=c["start_frame"] * fs,
                                    start_frame=c["start_frame"])
        kw = dict(current_start=c["start_frame"] * fs, start_frame=c["start_frame"], local_attn_size=W, sink_size=S,
                  text_len=g["text_len"])
        with torch.no_grad():
            yb = w8_ref.causal_model_w8(c["latents"], g["text"], c["timestep"], g["sd"], H, kb, xb, **kw)
            y32 = w8_ref.causal_model_w8(c["latents"].float(), g["text"].float(), c["timestep"], sd32, H, k32, x32, **kw)
        e, floor = assert_bf16_parity(y, y32, yb, name=f"int8w causal model call {i}")
        print(f"int8w causal model call {i}: relL2 {e:.3e} (floor {floor:.3e}); {rel_l2(y, c['y_ref_bf16']):.3e} from the bf16 "
              f"reference")
    assert kv[0].head != 0


# ------------------------------------------------------------------------------------------------ graph, memory, SP
def test_denoiser_graph_replay_bit_equal_w8(golden_dir):
    from fastvideo_b200.api import WanDenoiser
    g, cfg, model = _model(golden_dir, int8_weights=True)
    den = WanDenoiser(model, use_graph=True)
    lat = g["latents"].pin_memory()
    txt = g["text"].pin_memory()
    t = float(g["timestep"][0])
    out = den.step(lat, txt, t)
    torch.cuda.synchronize()
    assert den.graph_status == "captured", den.graph_status
    out = out.clone()
    eager = model.forward(g["latents"].cuda(), g["text"].cuda(), torch.full((1,), t, device="cuda"))
    assert torch.equal(out, eager.cpu())
    out2 = den.step(lat, txt, t)
    torch.cuda.synchronize()
    assert torch.equal(out2, out)


def _block_weight_bytes(blk):
    from fastvideo_b200 import ops
    total = 0
    for v in vars(blk).values():
        if isinstance(v, ops.Int8Weight):
            total += v.nbytes
        elif torch.is_tensor(v):
            total += v.numel() * v.element_size()
    return total


def test_14b_block_weight_bytes_halved():
    from fastvideo_b200 import wan_dit
    cfg = wan_dit.WanDiTConfig(**wan_dit.WAN_14B, vsa=True)
    sd = wan_dit.random_state_dict(wan_dit.WanDiTConfig(**{**cfg.__dict__, "num_layers": 1}), "cuda", layers=1)
    bf16 = _block_weight_bytes(wan_dit.WanBlock(sd, "blocks.0.", cfg))
    int8 = _block_weight_bytes(wan_dit.WanBlock(sd, "blocks.0.", wan_dit.WanDiTConfig(**wan_dit.WAN_14B, vsa=True,
                                                                                       int8_weights=True)))
    print(f"14B VSA block weights: bf16 {bf16 / 2**20:.1f} MiB, int8 {int8 / 2**20:.1f} MiB ({int8 / bf16:.3f}x)")
    assert int8 <= 0.51 * bf16


def test_sequence_parallel_and_causal_accept_int8_weights(golden_dir):
    """The sequence-parallel and causal classes take an int8_weights model (their fp8 / 8-bit attention refusals stay)."""
    from fastvideo_b200 import causal_wan, distributed
    g, cfg, model = _model(golden_dir, int8_weights=True)
    distributed.SPWanDiT(model, 0, 1)
    _, _, cmodel = _causal_model(golden_dir, True)
    causal_wan.SPCausalWanDiT(cmodel, 0, 1)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_sp_w8_equals_single_rank(tmp_path):
    """tests/sp_worker.py int8 on 2 ranks: SPWanDiT with int8_weights bit-equal to the single-rank engine (dense and VSA, push
    and NCCL), SPCausalWanDiT with int8_weights within bf16 rounding of it."""
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, {torch.cuda.device_count()} visible")
    out = str(tmp_path / f"sp_w8_parity_{world}.json")
    env = dict(os.environ, SP_WORKER_OUT=out)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "sp_worker.py"), "int8"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    assert p.returncode == 0, (p.stdout[-3000:], p.stderr[-3000:])
    res = json.load(open(out))
    assert any(r.get("causal") and "call" in r for r in res), res
    assert all(r["ok_all_ranks"] for r in res if "skipped" not in r), res
