"""CPU: every row-kernel entry point of csrc/elementwise.cu refuses a pointer that its kernels access with 16-byte vectors
when that pointer is 8 bytes off alignment (include/fvb200.h, "Row kernels"): FVB_ERR_INVALID_ARG, before any launch.

The calls run in a subprocess with CUDA_VISIBLE_DEVICES="" and fake device addresses that are never dereferenced. An entry
point that lost its check would then try to launch and return a CUDA error ("no device") instead of FVB_ERR_INVALID_ARG, so
the test fails without a misaligned kernel ever reaching a GPU. The same call with every pointer aligned must get past the
argument checks (a CUDA error, not FVB_ERR_INVALID_ARG): the refusal is then due to the one shifted pointer."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FVB_ERR_INVALID_ARG = 1

# (entry point, the pointers its kernels access with 16-byte vectors)
VECTOR_POINTERS = {
    "ln_mod": ["x", "out", "hidden_out", "w", "b", "scale", "shift"],
    "ln_mod_f32": ["x", "out", "w", "b"],
    "rmsnorm_rope": ["x0", "x1", "w0", "w1", "cos", "sin"],
    "rmsnorm_rope_f64": ["cos", "sin"],
    "rmsnorm_rope_scatter": ["x0", "x1", "y0", "y1", "w0", "w1", "cos", "sin"],
    "rmsnorm_bwd": ["x", "w", "dy", "dx", "ws"],
    "rmsnorm_rope_bwd": ["x0", "w0", "dy0", "dx0", "x1", "w1", "dy1", "dx1", "cos", "sin", "ws"],
    "bias_grad": ["dy", "ws"],
    "resid_gate_bwd": ["dout", "y", "gate", "dy", "ws"],
    "resid_gate_bwd_f32": ["dout"],
    "ln_mod_bwd": ["x", "dn", "gain", "gin", "dx", "ws"],
    "ln_mod_grouped_bwd": ["x", "dn", "scale", "gin", "dx", "ws"],
    "resid_gate_grouped_bwd": ["dout", "y", "gate", "dy", "ws"],
}

_CHILD = r"""
import json, sys
from ctypes import c_float, c_int, c_int64, c_void_p
from fastvideo_b200 import _lib

L = _lib.lib()
M, D, HD, WS = 600, 1536, 128, 1 << 30
spec = json.loads(sys.argv[1])
out = {}
for case, names in spec.items():
    for shifted in [None] + names:
        base = {}
        def P(name):
            # distinct fake device addresses, 4 KiB apart; the shifted one is 8 bytes off
            if name not in base:
                base[name] = (1 << 32) + 4096 * (len(base) + 1)
            return c_void_p(base[name] + (8 if name == shifted else 0))
        i, i64, f = c_int, c_int64, c_float
        s = c_void_p(0)
        if case in ("ln_mod", "ln_mod_f32"):
            f32 = case == "ln_mod_f32"
            rc = L.fvb_layernorm_modulate(P("x"), i(int(f32)), i64(D), P("w"), P("b"), None if f32 else P("scale"),
                                          None if f32 else P("shift"), i(0), i64(0), i(1), P("out"), i64(D),
                                          None if f32 else P("hidden_out"), i64(D), i(M), i(D), f(1e-6), s)
        elif case in ("rmsnorm_rope", "rmsnorm_rope_f64"):
            f64 = case == "rmsnorm_rope_f64"
            rc = L.fvb_rmsnorm_rope(P("x0"), P("w0"), i64(D), P("x1"), P("w1"), i64(D), P("cos"), P("sin"), i(int(f64)), None,
                                    None, i(M), i(D), i(HD), f(1e-6), s)
        elif case == "rmsnorm_rope_scatter":
            rc = L.fvb_rmsnorm_rope_scatter(P("x0"), P("w0"), i64(D), P("x1"), P("w1"), i64(D), P("y0"), P("y1"), i64(D),
                                            P("offsets"), P("cos"), P("sin"), i(0), None, i(M), i(D), i(HD), f(1e-6), s)
        elif case == "rmsnorm_bwd":
            rc = L.fvb_rmsnorm_bwd(P("x"), i64(D), P("w"), P("dy"), i64(D), P("dx"), i64(D), P("dw"), P("ws"), i64(WS), i(M),
                                   i(D), f(1e-6), s)
        elif case == "rmsnorm_rope_bwd":
            rc = L.fvb_rmsnorm_rope_bwd(P("x0"), i64(D), P("w0"), P("dy0"), i64(D), P("dx0"), i64(D), P("dw0"), P("x1"), i64(D),
                                        P("w1"), P("dy1"), i64(D), P("dx1"), i64(D), P("dw1"), P("cos"), P("sin"), None,
                                        P("ws"), i64(WS), i(M), i(D), i(HD), f(1e-6), s)
        elif case == "bias_grad":
            rc = L.fvb_bias_grad_bf16(P("dy"), i64(D), P("db"), P("ws"), i64(WS), i(M), i(D), s)
        elif case in ("resid_gate_bwd", "resid_gate_bwd_f32"):
            rc = L.fvb_resid_gate_bwd(P("dout"), i(int(case.endswith("f32"))), i64(D), P("y"), i64(D), P("gate"), P("dy"),
                                      i64(D), P("d_gate"), P("db"), P("ws"), i64(WS), i(M), i(D), s)
        elif case == "ln_mod_bwd":
            rc = L.fvb_layernorm_modulate_bwd(P("x"), i(0), i64(D), P("dn"), i64(D), P("gain"), i(1), i(1), P("gin"), i(0),
                                              i64(D), P("dx"), i64(D), P("d_gain"), P("d_offset"), P("ws"), i64(WS), i(M),
                                              i(D), f(1e-6), s)
        elif case == "ln_mod_grouped_bwd":
            rc = L.fvb_layernorm_modulate_grouped_bwd(P("x"), i64(D), P("dn"), i64(D), P("scale"), i(60), i64(D), P("gin"),
                                                      i(1), i64(D), P("dx"), i64(D), P("d_scale"), P("d_shift"), i64(D),
                                                      P("ws"), i64(WS), i(M), i(D), f(1e-6), s)
        elif case == "resid_gate_grouped_bwd":
            rc = L.fvb_resid_gate_grouped_bwd(P("dout"), i64(D), P("y"), i64(D), P("gate"), i(60), i64(D), P("dy"), i64(D),
                                              P("d_gate"), i64(D), P("db"), P("ws"), i64(WS), i(M), i(D), s)
        else:
            raise ValueError(case)
        out[f"{case}:{shifted}"] = [rc, L.fvb_last_error().decode(errors="replace")]
print(json.dumps(out))
"""


@pytest.fixture(scope="module")
def codes():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable, "-c", _CHILD, json.dumps(VECTOR_POINTERS)], capture_output=True, text=True,
                       timeout=300, cwd=ROOT, env=env)
    assert p.returncode == 0, p.stderr[-2000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", sorted(VECTOR_POINTERS))
def test_aligned_call_passes_the_argument_checks(codes, case):
    rc, msg = codes[f"{case}:None"]
    assert rc not in (0, FVB_ERR_INVALID_ARG), f"{case}: aligned arguments gave {rc} ({msg}); expected a no-device CUDA error"


@pytest.mark.parametrize("case", sorted(VECTOR_POINTERS))
def test_misaligned_pointer_is_refused(codes, case):
    for name in VECTOR_POINTERS[case]:
        rc, msg = codes[f"{case}:{name}"]
        assert rc == FVB_ERR_INVALID_ARG and "16-byte aligned" in msg, f"{case}: {name} 8 bytes off gave {rc} ({msg})"
