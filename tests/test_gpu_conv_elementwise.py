"""GPU: the Wan VAE decoder's implicit-GEMM convolution (csrc/conv3d_sm90.cu) element by element, through the C ABI
(tests/elementwise_ref.py, "Convolutions"): grid and tap-probe inputs bit for bit, random bf16 inputs against fp64 element
bounds, and the fused RMS norm (bf16 and e4m3 outputs) replayed bit for bit against the kernel's own raw output.

Outputs go into sentinel buffers: a gap after Cout in every row, an element before the first row. Inputs the kernel must not
read hold values that would show: the frame after t_off + T_out holds huge values, the weight columns past Cin hold
non-zero garbage (the input's channels past Cin must be zero-filled), the residual's row gaps and everything after bias,
w_scale and gamma hold NaN. `conv_path` mirrors conv3d_impl's choice of instantiation, so a CPU test can assert that the
case lists reach every one.

Results on an NVIDIA H100 80GB HBM3 at a 700 W power limit: every grid, tap-probe, dense e4m3 grid and fused-norm output
bit for bit (the e4m3 norm with SiLU inside its round-to-nearest interval), largest error / bound 0.9997 on random bf16
inputs. The random FP8 convolution has no element bound here: it needs a model of the e4m3 accumulator, which is
unpublished; the probes and the dense grid check its data movement instead, and tests/test_gpu_vae_fp8.py its accuracy."""
from ctypes import c_float, c_int, c_int64
import zlib

import pytest
import torch

import elementwise_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
NAN = float("nan")
FVB_ERR_INVALID_ARG = 1


# ------------------------------------------------------------------------------------------------ launch choices
def cin_pad_of(Cin):
    """ops.pack_conv_weight's channel padding: 64-channel k-blocks when possible, else 32."""
    return Cin if Cin % 64 == 0 else -(-Cin // 32) * 32


def conv_path(Cin, Cout, fp8, norm):
    """conv3d_impl's instantiation (fp8, BN, BK, NORM, KSUB) for a packed weight of Cin channels."""
    cp = cin_pad_of(Cin)
    BK = (128 if cp % 128 == 0 else 64 if cp % 64 == 0 else 32) if fp8 else (64 if cp % 64 == 0 else 32)
    BN = 192 if Cout > 128 else 128 if Cout > 96 else 96 if Cout > 16 else 16
    ksub_ok = BK < 128 if fp8 else (BK == 32 and BN <= 128)
    return (fp8, BN, BK, norm, 3 if ksub_ok and (cp // BK) % 3 == 0 else 1)


def conv_instantiations():
    """Every (fp8, BN, BK, NORM, KSUB) that conv3d_impl's dispatch and launch_conv can launch."""
    out = set()
    for fp8 in (False, True):
        for norm in (0, 1, 2):
            for BN in ((16, 96, 128, 192) if norm == 0 else (96, 128, 192)):
                for BK in ((32, 64, 128) if fp8 else (32, 64)):
                    out.add((fp8, BN, BK, norm, 1))
                    if (BK < 128) if fp8 else (BK == 32 and BN <= 128):
                        out.add((fp8, BN, BK, norm, 3))
    return out


# ------------------------------------------------------------------------------------------------ cases
def case(Cin, Cout, fp8=False, norm=0, k=(3, 3, 3), T_out=2, t_off=0, H=9, W=17, bias=True, resid=False, out_gap=8,
         out_off=1, resid_gap=8, norm_gap=16, silu=False, raw=True, bound0=False, interleave=0):
    """One convolution call. norm: 0 none, 1 bf16, 2 e4m3 normalised output. out_off: elements before the output's first
    row (1: 2-byte but not 4-byte aligned, the scalar-store path)."""
    return dict(Cin=Cin, Cout=Cout, fp8=fp8, norm=norm, k=k, T_out=T_out, t_off=t_off, H=H, W=W, bias=bias, resid=resid,
                out_gap=out_gap, out_off=out_off, resid_gap=resid_gap, norm_gap=norm_gap, silu=silu, raw=raw,
                bound0=bound0, interleave=interleave)


_CIN = {(False, 64, 1): [64, 40, 128], (False, 32, 1): [32, 16], (False, 32, 3): [96, 72],
        (True, 128, 1): [128, 256], (True, 64, 1): [64, 48], (True, 64, 3): [192], (True, 32, 1): [32], (True, 32, 3): [96]}
_COUT = {(16, 0): [16, 3, 8], (96, 0): [96, 17, 40], (128, 0): [97, 128], (192, 0): [129, 200, 192],
         (96, 1): [24, 96], (128, 1): [104, 128], (192, 1): [136, 192]}
_SPATIAL = [(1, 1), (7, 15), (8, 16), (9, 17), (7, 33), (9, 1), (1, 17), (8, 33)]
_TIME = [((3, 3, 3), 0, 3), ((3, 3, 3), 1, 2), ((3, 3, 3), 2, 1), ((1, 1, 1), 0, 2), ((3, 3, 3), 0, 4), ((1, 3, 3), 0, 2),
         ((3, 1, 1), 1, 2)]


def dispatch_cases():
    """One case (or more) per instantiation, rotating through the spatial, time and epilogue edges."""
    out = []
    i = 0
    for inst in sorted(conv_instantiations()):
        fp8, BN, BK, norm, ksub = inst
        cins = _CIN[(fp8, BK, ksub)]
        couts = _COUT[(BN, min(norm, 1))]
        for j in range(max(len(cins), len(couts)) if norm == 0 else 1):
            H, W = _SPATIAL[i % len(_SPATIAL)]
            k, t_off, T_out = _TIME[i % len(_TIME)]
            Cin, Cout = cins[j % len(cins)], couts[j % len(couts)]
            if norm:
                c = case(Cin, Cout, fp8, norm, k, T_out, t_off, max(H, 5), W, bias=i % 2 == 0, resid=i % 3 == 0,
                         out_gap=8 * (i % 2), out_off=0, resid_gap=8 * (i % 2), norm_gap=16 * (i % 2), silu=i % 2 == 1,
                         raw=i % 3 != 1)
            else:
                c = case(Cin, Cout, fp8, 0, k, T_out, t_off, H, W, bias=i % 2 == 0, resid=i % 3 == 0,
                         out_gap=(0, 8, 5)[i % 3], out_off=i % 2, resid_gap=(3, 0, 8)[i % 3])
            assert conv_path(Cin, Cout, fp8, norm) == inst
            out.append(c)
            i += 1
    return out


DISPATCH_CASES = dispatch_cases()

EDGE_CASES = [
    case(64, 216, H=9, W=33, resid=True),  # two N blocks, the second partial (24 of 192 columns)
    case(384, 384, k=(3, 3, 3), T_out=2, t_off=1, H=8, W=16, resid=True),
    case(128, 576, fp8=True, k=(1, 3, 3), T_out=1, H=7, W=17, resid=True, resid_gap=8),  # bias / w_scale at n >= 512: global
    case(64, 576, k=(1, 1, 1), T_out=1, H=9, W=15, bias=True),
    case(96, 3, H=9, W=33, out_gap=0),  # conv_out: Cout = 3, odd out_ld, scalar stores
    case(96, 3, fp8=True, H=8, W=16, out_gap=0, out_off=0),
    case(32, 64, k=(3, 1, 1), T_out=2, t_off=1, H=9, W=17, bias=True, interleave=32),  # WanResample time_conv
    case(64, 128, k=(3, 1, 1), T_out=3, t_off=0, H=8, W=16, interleave=64, out_off=0),
    case(384, 768, k=(3, 1, 1), T_out=2, t_off=2, H=7, W=15, interleave=384, out_gap=8),  # real width: bias >= 512 global
    case(96, 96, k=(3, 3, 3), T_out=4, t_off=0, H=9, W=33, resid=True),  # dt_first 2, 1, 0, 0
    case(96, 96, fp8=True, k=(3, 3, 3), T_out=4, t_off=0, H=9, W=17, resid=True, out_off=0),
]

NORM_CASES = [
    case(Cin, Cout, fp8, norm, (3, 3, 3), 2, t_off, 9, 17, bias=True, resid=resid, out_gap=8, out_off=0, resid_gap=8,
         norm_gap=16, silu=silu, raw=raw, bound0=bound0)
    for (Cin, Cout, fp8, norm, t_off, resid, silu, raw, bound0) in [
        (64, 24, False, 1, 0, True, False, True, False), (96, 96, False, 1, 1, False, True, False, False),
        (64, 128, False, 2, 2, True, False, True, False), (128, 136, False, 2, 0, False, True, False, False),
        (96, 192, False, 1, 1, True, False, False, False), (96, 96, True, 2, 0, True, False, True, False),
        (192, 192, True, 2, 1, False, True, True, False), (128, 136, True, 1, 2, True, False, False, False),
        (64, 24, True, 1, 0, False, True, True, False), (128, 128, True, 2, 0, True, True, False, False),
        (96, 96, False, 2, 0, True, False, True, True), (96, 96, True, 2, 1, False, True, False, True)]]

# At least one full-resolution frame per decoder width: more tiles than SMs and not a multiple of them, frames of different
# k-block counts (t_off 0: frame 0 reads one time tap, frame 1 two), so a CTA's next tile starts mid-ring with another nkb.
PERSISTENT_CASES = [case(96, 96, H=480, W=832, resid=True, out_off=0), case(96, 3, H=480, W=832, out_gap=0),
                    case(192, 192, H=240, W=416, resid=True, out_off=0), case(384, 384, H=120, W=208, out_off=0),
                    case(192, 192, fp8=True, H=240, W=416, resid=True, out_off=0)]


def case_id(c):
    s = f"{'e4m3' if c['fp8'] else 'bf16'}-{c['Cin']}x{c['Cout']}-k{''.join(map(str, c['k']))}-T{c['T_out']}o{c['t_off']}"
    s += f"-{c['H']}x{c['W']}"
    for key, tag in (("bias", "b"), ("resid", "r"), ("silu", "silu"), ("bound0", "q0")):
        s += f"-{tag}" if c[key] else ""
    if c["norm"]:
        s += f"-norm{c['norm']}" + ("-raw" if c["raw"] else "")
    if c["interleave"]:
        s += f"-il{c['interleave']}"
    return s + f"-ld{c['out_gap']}+{c['out_off']}"


# ------------------------------------------------------------------------------------------------ buffers
def _abi():
    from fastvideo_b200 import _lib
    return _lib.lib(), _lib.check, _lib.ptr, _lib.stream_ptr


def _gen(*key):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


class Rows:
    """A [F, H, W, C] view with row stride ld = C + gap, `off` elements into a sentinel buffer with 64 spare elements."""

    def __init__(self, F, H, W, C, gap, off, dtype, seed):
        self.ld = C + gap
        n = off + F * H * W * self.ld + 64
        self.g = R.Guarded((n,), dtype, DEV, seed=seed)
        self.v = self.g.region(torch.as_strided(self.g.buf, (F, H, W, C), (H * W * self.ld, W * self.ld, self.ld, 1), off))


def _nan_after(t, extra=64):
    """t (1-D) followed by NaN in the same allocation."""
    buf = torch.full((t.numel() + extra,), NAN, dtype=t.dtype, device=DEV)
    buf[:t.numel()] = t
    return buf[:t.numel()]


def _strided(t, gap, fill):
    """t [T, H, W, C] in a buffer of row stride C + gap whose gaps hold `fill`."""
    buf = torch.full((*t.shape[:-1], t.shape[-1] + gap), fill, dtype=t.dtype, device=DEV)
    buf[..., :t.shape[-1]] = t
    return buf[..., :t.shape[-1]]


def inputs(c, kind):
    """Operands of one case: kind "grid" (bf16 grid / dense e4m3 grid), "probe" or "random" (bf16 only). Returns a dict
    with x [T_in, H, W, Cin] and w [Cout, ntaps, Cin_pad] in the kernel's dtype, their float values, bias, resid,
    w_scale, x_scale, the exactness quantum (None: random)."""
    g = _gen("conv", case_id(c), kind)
    Cin, Cout, (kt, kh, kw), T_out, t_off = c["Cin"], c["Cout"], c["k"], c["T_out"], c["t_off"]
    ntaps, cp = kt * kh * kw, cin_pad_of(Cin)
    T_in = t_off + T_out + 1
    shape = (T_in, c["H"], c["W"], Cin)
    Cres = Cout
    if kind == "grid" and c["fp8"]:
        x, w = R.fp8_dense_grid(shape, Cout, ntaps, Cin, cp, g, DEV)
        quantum = 1.0
    elif kind == "probe":
        x = torch.randint(-7, 8, shape, generator=g, device=DEV).float()
        w = R.probe_weights(Cout, ntaps, Cin, cp, g, DEV)
        quantum = 1.0
    elif kind == "grid":
        x, w = R.grid_bf16(shape, g, DEV).float(), R.grid_bf16((Cout, ntaps, cp), g, DEV).float()
        quantum = 2.0 ** -8
    else:
        x = torch.randn(shape, generator=g, device=DEV)
        w = torch.randn(Cout, ntaps, cp, generator=g, device=DEV) / (ntaps * Cin) ** 0.5
        quantum = None
    dt = torch.float8_e4m3fn if c["fp8"] else torch.bfloat16
    x, w = x.to(dt).clone(), w.to(dt).clone()
    x[t_off + T_out:] = 448.0 if c["fp8"] else 2.0 ** 100  # never read
    if cp > Cin:  # garbage weights on channels the input's zero fill must cancel
        w[:, :, Cin:] = (torch.randint(0, 2, (Cout, ntaps, cp - Cin), generator=g, device=DEV).float() * 2 - 1).to(dt)
    small = lambda *s: (R.grid_bf16(s, g, DEV) if quantum else R.rand_bf16(s, g, DEV, 0.5))
    bias = _nan_after(small(Cout)) if c["bias"] else None
    resid = _strided(small(T_out, c["H"], c["W"], Cres), c["resid_gap"], NAN) if c["resid"] else None
    w_scale = x_scale = None
    if c["fp8"]:
        w_scale = _nan_after(torch.rand(Cout, generator=g, device=DEV) * 0.05 + 0.01)
        x_scale = R.f32(0.0371)
    return dict(x=x.contiguous(), w=w.contiguous(), bias=bias, resid=resid, w_scale=w_scale, x_scale=x_scale,
                quantum=quantum, cp=cp, T_in=T_in)


def call_conv(c, d, out, out_ld, norm_out=None, norm_ld=0, gamma=None, bound=0.0):
    """The entry point of the case (plain when norm_out is None); returns the status code."""
    L, _, ptr, sp = _abi()
    Cin, Cout, (kt, kh, kw) = c["Cin"], c["Cout"], c["k"]
    x, w, cp = d["x"], d["w"], d["cp"]
    resid, rld = d["resid"], c["Cout"] + c["resid_gap"]
    T_in, H, W = d["T_in"], c["H"], c["W"]
    head = (ptr(x), c_int(T_in), c_int(H), c_int(W), c_int(Cin))
    mid = (c_int(kt), c_int(kh), c_int(kw), ptr(d["bias"]), ptr(resid), c_int64(rld if resid is not None else 0), ptr(out),
           c_int64(out_ld), c_int(c["T_out"]), c_int(c["t_off"]))
    if c["fp8"]:
        wpart = (c_float(d["x_scale"]), ptr(w), ptr(d["w_scale"]), c_int(cp), c_int(Cout))
        if norm_out is None:
            return L.fvb_conv3d_cl_fp8(*head, *wpart, *mid, sp())
        return L.fvb_conv3d_cl_fp8_norm(*head, *wpart, *mid, ptr(gamma), ptr(norm_out), c_int64(norm_ld),
                                        c_int(int(c["silu"])), c_int(int(c["norm"] == 2)), c_float(bound), sp())
    wpart = (ptr(w), c_int(cp), c_int(Cout))
    if norm_out is None:
        return L.fvb_conv3d_cl(*head, *wpart, *mid, c_int(c["interleave"]), sp())
    if c["norm"] == 1:
        return L.fvb_conv3d_cl_norm(*head, *wpart, *mid, ptr(gamma), ptr(norm_out), c_int64(norm_ld), c_int(int(c["silu"])),
                                    sp())
    return L.fvb_conv3d_cl_norm_e4m3(*head, *wpart, *mid, ptr(gamma), ptr(norm_out), c_int64(norm_ld), c_int(int(c["silu"])),
                                     c_float(bound), sp())


def conv_ref(c, d, kind):
    """(exact bf16 output, None) for the exact kinds, (fp64 reference, bound) for random; [T_out, H, W, Cout]."""
    e, A = R.conv_exact(d["x"].float(), d["w"].float(), c["k"], c["T_out"], c["t_off"])
    if d["quantum"] is not None:
        R.assert_conv_exact_premise(A, d["quantum"], case_id(c))
        if kind == "grid" and c["fp8"]:  # integers below 2^11: exact on an accumulator of >= 12 bits
            assert float(A.max()) <= 2048
        resid = d["resid"]
        return R.conv_epilogue_ref(e.float(), d["bias"], resid, d["x_scale"], d["w_scale"]), None
    K = max(R.conv_k_read(c["k"], d["cp"], c["T_out"], c["t_off"]))
    return R.conv_bound(e, A, K, d["bias"], d["resid"])


def family(c, kind):
    if kind == "probe":
        return f"conv {'e4m3' if c['fp8'] else 'bf16'} tap probes"
    if kind == "grid":
        return "conv e4m3 dense grid (>= 12-bit accumulator)" if c["fp8"] else "conv bf16 (grid inputs)"
    return "conv bf16 (random)"


def run_plain(c, kind, seed=1):
    """Run the plain convolution of a case into a sentinel buffer, check it; returns (inputs, out view, reference)."""
    d = inputs(c, kind)
    _, check, _, _ = _abi()
    il = c["interleave"]
    F, Cw = (2 * c["T_out"], il) if il else (c["T_out"], c["Cout"])
    o = Rows(F, c["H"], c["W"], Cw, c["out_gap"], c["out_off"], torch.bfloat16, seed)
    check(call_conv(c, d, o.v, o.ld))
    torch.cuda.synchronize()
    o.g.assert_untouched(f"{case_id(c)} out")
    ref, bound = conv_ref(c, d, kind)
    got = o.v
    if il:  # output channel n goes to frame 2 t + n / il, channel n % il
        got = torch.cat([o.v[0::2], o.v[1::2]], -1)
    BN = conv_path(c["Cin"], c["Cout"], c["fp8"], 0)[1]
    where = lambda i: R.conv_coords(i, BN)
    if bound is None:
        R.assert_exact(got, ref, f"{case_id(c)} {kind}", where, family=family(c, kind))
    else:
        R.assert_within(got, ref, bound, f"{case_id(c)} {kind}", where, family=family(c, kind))
    return d, o, ref


def _kinds(c):
    return ["grid", "probe"] if c["fp8"] else ["grid", "random", "probe"]


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    R.print_summary(request.config)
    name = torch.cuda.get_device_name(0)
    try:
        import subprocess
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    cap = request.config.pluginmanager.getplugin("capturemanager")
    if cap is not None:
        with cap.global_and_fixture_disabled():
            print(f"  device: {name}, power limit {pl}", flush=True)


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("c", [c for c in DISPATCH_CASES if c["norm"] == 0] + EDGE_CASES, ids=case_id)
def test_conv_plain(c):
    for kind in _kinds(c):
        run_plain(c, kind)


def _norm_gap(c):
    """norm_out's row gap: norm_gap, plus what makes an e4m3 row stride a multiple of 16 bytes."""
    return c["norm_gap"] + ((-c["Cout"]) % 16 if c["norm"] == 2 else 0)


def check_norm(c, y, gamma, got, bound, name):
    """The fused norm's output got [.., Cout] (bf16 or e4m3) against the replay on the raw output y."""
    Cout = c["Cout"]
    v = R.conv_norm_replay(y.reshape(-1, Cout), gamma, Cout)
    got = got.reshape(-1, Cout)
    qs = R.e4m3_qscale(bound) if c["norm"] == 2 else None
    fam = f"conv fused norm {'e4m3' if c['norm'] == 2 else 'bf16'} out"
    if not c["silu"]:
        if c["norm"] == 2:
            R.assert_exact(got.view(torch.uint8), R.e4m3_code(v, qs).view(torch.uint8), name, family=fam)
        else:
            R.assert_exact(got, v.bfloat16(), name, family=fam)
        return
    ref, b = R.silu_bound(v)
    R.assert_rounds_from(got.float(), ref, b, name, qscale=qs, family=fam + " (SiLU, round-to-nearest interval)")


@pytest.mark.parametrize("c", [c for c in DISPATCH_CASES if c["norm"]] + NORM_CASES, ids=case_id)
def test_conv_fused_norm(c):
    _, check, _, _ = _abi()
    Cout = c["Cout"]
    for kind in _kinds(c):
        d, plain, _ = run_plain(c, kind)
        g = _gen("gamma", case_id(c), kind)
        gamma = _nan_after(1 + 0.2 * torch.randn(Cout, generator=g, device=DEV))
        bound = 0.0 if c["bound0"] else R.f32(float(torch.tensor(float(Cout)).sqrt() * gamma.abs().max().cpu()))
        ndt = torch.float8_e4m3fn if c["norm"] == 2 else torch.bfloat16
        shp = (c["T_out"], c["H"], c["W"], Cout)
        raw = Rows(*shp, c["out_gap"], 0, torch.bfloat16, 2) if c["raw"] else None
        nout = Rows(*shp, _norm_gap(c), 0, ndt, 3)
        check(call_conv(c, d, raw.v if raw else None, raw.ld if raw else Cout, nout.v, nout.ld, gamma, bound))
        torch.cuda.synchronize()
        nout.g.assert_untouched(f"{case_id(c)} norm_out")
        if raw:
            raw.g.assert_untouched(f"{case_id(c)} raw out")
            R.assert_exact(raw.v, plain.v, f"{case_id(c)} raw vs plain conv", family="conv fused norm raw out")
        check_norm(c, plain.v, gamma, nout.v, bound, f"{case_id(c)} {kind} norm")


@pytest.mark.parametrize("c", PERSISTENT_CASES, ids=case_id)
def test_conv_persistent_walk(c):
    tiles = -(-c["W"] // 16) * -(-c["H"] // 8) * c["T_out"] * -(-c["Cout"] // conv_path(c["Cin"], c["Cout"], c["fp8"], 0)[1])
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert tiles > sms and tiles % sms != 0
    for kind in (["grid"] if c["fp8"] else ["grid", "random"]):
        run_plain(c, kind)
        torch.cuda.empty_cache()


def test_conv_refused_calls_write_nothing():
    """Argument checks return FVB_ERR_INVALID_ARG before any launch: the output buffers keep their bits."""
    torch.cuda.synchronize()
    cases = [
        (case(64, 200, norm=1), {}),  # fused norm needs one N block (Cout <= 192)
        (case(64, 96, norm=1), {"norm_off": 4}),  # norm_out 8 bytes off 16-byte alignment
        (case(40, 64, fp8=True), {}),  # FP8 needs Cin % 16 == 0
        (case(32, 64, k=(3, 1, 1), resid=True, interleave=32, out_off=0), {}),  # interleave with a residual
    ]
    for c, opt in cases:
        d = inputs(c, "grid") if not (c["fp8"] and c["Cin"] % 16) else _fp8_any(c)
        o = Rows(c["T_out"] * (2 if c["interleave"] else 1), c["H"], c["W"], c["interleave"] or c["Cout"], 8, 0,
                 torch.bfloat16, 4)
        o.g.mask.zero_()  # nothing may be written at all
        nout = gamma = None
        if c["norm"]:
            nout = R.Guarded((opt.get("norm_off", 0) + c["T_out"] * c["H"] * c["W"] * c["Cout"] + 64,), torch.bfloat16, DEV)
            gamma = torch.ones(c["Cout"], device=DEV)
            nv = nout.buf[opt.get("norm_off", 0):]
        code = call_conv(c, d, o.v, o.ld, nv if c["norm"] else None, c["Cout"], gamma)
        torch.cuda.synchronize()
        assert code == FVB_ERR_INVALID_ARG, (case_id(c), code)
        o.g.assert_untouched(f"refused {case_id(c)}")
        if nout is not None:
            nout.assert_untouched(f"refused {case_id(c)} norm_out")


def _fp8_any(c):
    """FP8 operands for a shape the host refuses (Cin % 16 != 0): any bytes."""
    cp = cin_pad_of(c["Cin"])
    ntaps = c["k"][0] * c["k"][1] * c["k"][2]
    return dict(x=torch.zeros(c["t_off"] + c["T_out"] + 1, c["H"], c["W"], c["Cin"], dtype=torch.float8_e4m3fn, device=DEV),
                w=torch.zeros(c["Cout"], ntaps, cp, dtype=torch.float8_e4m3fn, device=DEV), bias=None, resid=None,
                w_scale=torch.ones(c["Cout"], device=DEV), x_scale=1.0, quantum=1.0, cp=cp,
                T_in=c["t_off"] + c["T_out"] + 1)


def test_conv_checkers_reject_mutants_of_real_output():
    """Each defect, edited into a copy of a passing kernel output, fails its checker."""
    c = case(64, 216, H=9, W=33, resid=True, out_off=0)
    d, o, ref = run_plain(c, "grid")
    got = o.v.clone()

    def rejected(mut, name):
        with pytest.raises(AssertionError):
            R.assert_exact(mut, ref, name)

    # one tap dropped in a border tile: tile (1, 2) (rows 8.., columns 32..) without tap (dt 2, dh 0, dw 0)
    xf, wf = d["x"].float(), d["w"].float().clone()
    wf[:, 18] = 0
    e2, _ = R.conv_exact(xf, wf, c["k"], c["T_out"], c["t_off"], want_abs=False)
    m = got.clone()
    m[:, 8:, 32:] = R.conv_epilogue_ref(e2.float(), d["bias"], d["resid"])[:, 8:, 32:]
    rejected(m, "tap dropped")
    # one tile's halo shifted by a pixel: tile (0, 1) computed from the input moved one column left
    e3, _ = R.conv_exact(torch.roll(xf, 1, 2), d["w"].float(), c["k"], c["T_out"], c["t_off"], want_abs=False)
    m = got.clone()
    m[:, :8, 16:32] = R.conv_epilogue_ref(e3.float(), d["bias"], d["resid"])[:, :8, 16:32]
    rejected(m, "halo shifted")
    # two 8-column groups swapped in the second N block
    m = got.clone()
    m[..., 192:200], m[..., 200:208] = got[..., 200:208], got[..., 192:200]
    rejected(m, "column groups swapped")
    # one byte past Cout
    o.g.buf.view(torch.uint8)[2 * (c["Cout"] + 1)] ^= 1
    with pytest.raises(AssertionError):
        o.g.assert_untouched("byte past Cout")
    # bias column n - 512 for n >= 512
    c = case(64, 576, k=(1, 1, 1), T_out=1, H=9, W=15, out_off=0)
    d, o, ref = run_plain(c, "grid")
    e, _ = R.conv_exact(d["x"].float(), d["w"].float(), c["k"], c["T_out"], c["t_off"], want_abs=False)
    wrong_bias = torch.cat([d["bias"][:512], d["bias"][:64]])
    rejected(R.conv_epilogue_ref(e.float(), wrong_bias, None), "bias n - 512")
    # interleave frames swapped
    c = case(32, 64, k=(3, 1, 1), T_out=2, t_off=1, H=9, W=17, interleave=32, out_off=0)
    d, o, ref = run_plain(c, "grid")
    m = torch.cat([o.v[1::2], o.v[0::2]], -1)
    rejected(m, "interleave frames swapped")
    # the norm: one e4m3 code one step off, and sqrt(BN) in place of sqrt(Cout)
    c = case(96, 104, norm=2, H=9, W=17, out_off=0)
    d, plain, _ = run_plain(c, "grid")
    gamma = _nan_after(1 + 0.2 * torch.randn(c["Cout"], generator=_gen("mut"), device=DEV))
    bound = R.f32(float(torch.tensor(104.0).sqrt() * gamma.abs().max().cpu()))
    nout = Rows(c["T_out"], c["H"], c["W"], 104, _norm_gap(c), 0, torch.float8_e4m3fn, 3)
    _abi()[1](call_conv(c, d, None, 104, nout.v, nout.ld, gamma, bound))
    torch.cuda.synchronize()
    check_norm(c, plain.v, gamma, nout.v, bound, "norm e4m3")
    m = nout.v.clone()
    m.view(torch.uint8)[0, 3, 5, 7] += 1
    with pytest.raises(AssertionError):
        check_norm(c, plain.v, gamma, m, bound, "one code one step off")
    v = R.conv_norm_replay(plain.v.reshape(-1, 104), gamma, 104, sqrt_of=128)
    with pytest.raises(AssertionError):
        R.assert_exact(nout.v.reshape(-1, 104).view(torch.uint8), R.e4m3_code(v, R.e4m3_qscale(bound)).view(torch.uint8),
                       "sqrt(BN)")
