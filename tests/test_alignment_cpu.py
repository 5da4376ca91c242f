"""CPU-only check that the vectorised entry points refuse a misaligned tensor base with an error return.

These kernels move 16 bytes per access.  A legal C-ABI call whose tensor starts mid-row (a column view) must come back
as a non-zero return with a message, not reach the device as a misaligned-address fault.  The calls run in a
subprocess that sees no CUDA device and pass fake, deliberately misaligned addresses with valid sizes: the alignment
check has to answer before any device work, and without it the call fails on the missing device with a different
message instead (nothing can launch, so nothing can fault)."""

import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_SCRIPT = r"""
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from pytorch_generative_b200 import _lib as L

lib = L.load()
A = 0x10000           # a fake 16-byte aligned device address
M = A + 8             # 8 bytes in: an fp32 column view starting at column 2, a bf16 one at column 4
taps_arr = (ctypes.c_int * 1)(0)
taps = ctypes.cast(taps_arr, ctypes.c_void_p)
calls = {
    "pg_act_cast_bf16": lambda: lib.pg_act_cast_bf16(M, 1, 8, 4, 8, L.ACT_RELU, A, 8, None),
    "pg_act_cast_bf16(out)": lambda: lib.pg_act_cast_bf16(A, 0, 8, 4, 8, L.ACT_RELU, M, 8, None),
    "pg_dact_from_out": lambda: lib.pg_dact_from_out(M, 1, A, 64, L.ACT_ELU, A, None),
    "pg_dact_from_out(ya)": lambda: lib.pg_dact_from_out(A, 0, M, 64, L.ACT_RELU, A, None),
    "pg_gated_act_fwd": lambda: lib.pg_gated_act_fwd(M, 0, 4, 8, L.ACT_TANH, A, 1, None),
    "pg_gated_act_bwd": lambda: lib.pg_gated_act_bwd(A, 0, M, 1, 4, 8, L.ACT_TANH, A, 0, None),
    "pg_gated_res_fwd": lambda: lib.pg_gated_res_fwd(A, 0, M, 4, 8, L.ACT_NONE, A, None),
    "pg_layernorm_fwd": lambda: lib.pg_layernorm_fwd(M, A, A, 4, 128, 1e-5, None, A, A, A, None),
    "pg_layernorm_bwd": lambda: lib.pg_layernorm_bwd(None, A, A, A, A, A, 4, 128, M, None, A, None, None, None, None, None),
    "pg_tap_gather": lambda: lib.pg_tap_gather(M, 8, 1, 2, 2, 8, 1, taps, taps, L.ACT_NONE, A, None),
    "pg_tap_scatter": lambda: lib.pg_tap_scatter(A, 1, 2, 2, 8, 1, taps, taps, L.ACT_NONE, None, 0, None, M, 8, None),
}
out = {}
for name, call in calls.items():
    rc = call()
    out[name] = [rc, lib.pg_last_error().decode(errors="replace")]
print(json.dumps(out))
"""

ENTRIES = ["pg_act_cast_bf16", "pg_act_cast_bf16(out)", "pg_dact_from_out", "pg_dact_from_out(ya)", "pg_gated_act_fwd",
           "pg_gated_act_bwd", "pg_gated_res_fwd", "pg_layernorm_fwd", "pg_layernorm_bwd", "pg_tap_gather",
           "pg_tap_scatter"]


@pytest.fixture(scope="module")
def results():
    from pytorch_generative_b200 import _build

    _build.build(verbose=False)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    proc = subprocess.run([sys.executable, "-c", _SCRIPT, ROOT], env=env, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stderr[-4000:]
    return json.loads(proc.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("entry", ENTRIES)
def test_misaligned_base_is_an_error(results, entry):
    rc, msg = results[entry]
    assert rc != 0 and "align" in msg, f"{entry}: rc={rc} message={msg!r}"
