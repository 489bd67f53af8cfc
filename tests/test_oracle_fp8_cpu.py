"""CPU: the FP8 restatement (tests/fp8_ref.py): the e4m3 row quantiser on hand-checked values, and which linears of the
Wan block restatement it runs in FP8.

e4m3fn: 1 sign, 4 exponent (bias 7), 3 mantissa bits; largest finite 448 (0x7e); subnormals m * 2^-9, m = 1..7. A row whose
amax is 448 has inv = 448 / 448 = 1 exactly, so its elements are converted unscaled and the rounding can be read off."""
import torch

import fp8_ref


def q_row(values, amax=448.0):
    x = torch.tensor([[amax] + list(values)], dtype=torch.float32).bfloat16()
    q, s = fp8_ref.quantize_fp8_rows(x)
    return q.view(torch.uint8)[0, 1:].tolist(), q.float()[0, 1:].tolist(), float(s[0])


def test_ties_round_to_even():
    # between 1.0 (0x38, mantissa 000) and 1.125 (0x39): the tie 1.0625 goes to the even 1.0;
    # between 1.125 and 1.25 (0x3a): the tie 1.1875 goes to the even 1.25; off-tie values go to the nearest
    bits, vals, s = q_row([1.0625, 1.1875, -1.0625, 1.09375])
    assert s == 1.0
    assert bits == [0x38, 0x3a, 0xb8, 0x39]
    assert vals == [1.0, 1.25, -1.0, 1.125]


def test_saturation_at_448():
    # 448 / amax * amax rounds above 448 for some amax: the element equal to amax must still give +-448, never NaN
    found = 0
    for a in torch.linspace(1.0, 1000.0, 4001).bfloat16().float().unique().tolist():
        inv = torch.tensor(448.0) / torch.tensor(a)
        if float(torch.tensor(a) * inv) > 448.0:
            x = torch.tensor([[a, -a, a / 2]]).bfloat16()
            q, s = fp8_ref.quantize_fp8_rows(x)
            assert q.view(torch.uint8)[0, :2].tolist() == [0x7e, 0xfe], a
            found += 1
    assert found > 0
    # and an element already at +-448 after scaling maps to the largest finite code
    bits, vals, _ = q_row([-448.0, 440.0])
    assert bits == [0xfe, 0x7e] and vals == [-448.0, 448.0]


def test_subnormals():
    # 2^-9 is the smallest subnormal (0x01); 1.5 * 2^-9 ties between 1 and 2 units -> 2 (0x02); 0.5 * 2^-9 ties between 0 and 1
    # unit -> 0; 0.75 * 2^-9 -> 1 unit; 7 * 2^-9 is the largest subnormal (0x07); 2^-6 is the smallest normal (0x08)
    u = 2.0 ** -9
    bits, vals, _ = q_row([u, 1.5 * u, 0.5 * u, 0.75 * u, 7 * u, 2.0 ** -6, -u])
    assert bits == [0x01, 0x02, 0x00, 0x01, 0x07, 0x08, 0x81]
    assert vals == [u, 2 * u, 0.0, u, 7 * u, 2.0 ** -6, -u]


def test_zero_row():
    x = torch.zeros(3, 40, dtype=torch.bfloat16)
    x[1, 5] = 0.5
    q, s = fp8_ref.quantize_fp8_rows(x)
    assert s[0] == 1.0 and s[2] == 1.0
    assert (q.view(torch.uint8)[0] == 0).all() and (q.view(torch.uint8)[2] == 0).all()
    assert s[1] == torch.tensor(0.5) / torch.tensor(448.0)
    assert q.float()[1, 5] == 448.0


def test_outlier_row():
    # amax 1000: inv = fp32(448 / 1000) = 0.448; the ones land on 0.448 -> 0.4375 (0.25 * (1 + 6/8), step 2^-5), the
    # outlier on 448, and the scale is fp32(1000 / 448)
    x = torch.ones(1, 64, dtype=torch.bfloat16)
    x[0, 17] = 1000.0
    q, s = fp8_ref.quantize_fp8_rows(x)
    inv = torch.tensor(448.0) / torch.tensor(1000.0)
    assert float(inv) == float(torch.tensor(0.448, dtype=torch.float32))
    assert q.float()[0, 17] == 448.0
    others = torch.cat([q.float()[0, :17], q.float()[0, 18:]])
    assert (others == 0.4375).all()
    assert s[0] == torch.tensor(1000.0) / torch.tensor(448.0)
    # the dequantised row: the ones come back within e4m3's relative step
    deq = (q.float() * s[:, None])[0]
    assert ((torch.cat([deq[:17], deq[18:]]) - 1.0).abs() < 2 ** -4).all()


def test_fp8_linear_restatement_is_exact_in_fp64():
    g = torch.Generator().manual_seed(7)
    x = torch.randn(5, 300, generator=g).bfloat16()
    w = torch.randn(24, 300, generator=g).bfloat16()
    xq, xs = fp8_ref.quantize_fp8_rows(x)
    wq, ws = fp8_ref.quantize_fp8_rows(w)
    y, exact = fp8_ref.fp8_linear_f32(xq, xs, wq, ws)
    # the dequantised operands reproduce the inputs to e4m3 precision, and the product to a few per cent
    assert torch.allclose(xq.float() * xs[:, None], x.float(), rtol=2 ** -4, atol=xs.max().item() * 2 ** -9)
    ref = x.float() @ w.float().t()
    assert float((y - ref).norm() / ref.norm()) < 5e-2
    assert float((y.double() - exact).abs().max()) <= float(exact.abs().max()) * 2 ** -20


def test_block_restatement_runs_exactly_the_token_stream_linears_in_fp8(monkeypatch):
    """wan_block_fp8 runs exactly the token-stream linears the engine quantises in FP8 -- the text-side K/V projections stay
    bf16 -- and leaves oracle/wan_ref as it found it."""
    from oracle import wan_ref
    from oracle.gen_golden import _rand_block_sd
    g = torch.Generator().manual_seed(3)
    D, H, L, seq = 256, 2, 8, (1, 2, 4)
    sd = _rand_block_sd(D, 512, H, True, g)
    x = torch.randn(1, 8, D, generator=g).bfloat16()
    ctx = torch.randn(1, L, D, generator=g).bfloat16()
    temb6 = (torch.randn(1, 6, D, generator=g) * 0.5).bfloat16()
    cos, sin = wan_ref.rotary_tables(seq, [44, 42, 42])
    seen = []
    real = fp8_ref.linear_fp8
    monkeypatch.setattr(fp8_ref, "linear_fp8", lambda x_, w, b: (seen.append(w), real(x_, w, b))[1])
    bf16_linear = wan_ref.linear
    with torch.no_grad():
        y8 = fp8_ref.wan_block_fp8(x, ctx, temb6, sd, "", H, cos, sin, attn_fn=wan_ref.sdpa)
        y16 = wan_ref.wan_block(x, ctx, temb6, sd, "", H, cos, sin, attn_fn=wan_ref.sdpa)
    assert wan_ref.linear is bf16_linear
    names = {k for k, v in sd.items() if any(v is w for w in seen)}
    assert names == {n + ".weight" for n in ("to_q", "to_k", "to_v", "to_out", "attn2.to_q", "attn2.to_out", "ffn.fc_in",
                                              "ffn.fc_out")}, names
    # the gate projection is a token-stream linear too, but the dense block (no vsa_meta) does not run it
    rel = float((y8.float() - y16.float()).norm() / y16.float().norm())
    assert 1e-3 < rel < 1e-1, rel
