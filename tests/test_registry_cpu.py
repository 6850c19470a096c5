"""The registry plumbing of an 8th backend (SURVEY.md 8b): tools/gen_backend_ph.py re-derives the reference's perfect hashes
(lib/nnc/cmd/build-cmd.rb:303-386, lib/nnc/cmd/ccv_nnc_cmd.inc:152-190) and the stand-alone host dispatches through
init_map[_ccv_nnc_cmd_ph(cmd)].backends[_ccv_nnc_cmd_backend_ph(backend)] exactly as lib/nnc/ccv_nnc_cmd.c does."""
import json
import os
import subprocess
import sys

import pytest

from ccv_b200 import abi, nnc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the reference's generated registry tables (lib/nnc/cmd/ccv_nnc_cmd.inc), extracted by tests/golden/make_golden.py
REGISTRY = os.path.join(ROOT, "tests", "golden", "reference_cmd_registry.json")
REFERENCE_BACKENDS = {"CPU_OPT": 0x46deb194, "CPU_REF": 0x3d9883e5, "GPU_CUBLAS": 0x9b8cfed, "GPU_CUDNN": 0x854b679a, "GPU_NCCL": 0x7afed9c7, "GPU_REF": 0x5f19790a, "MPS": 0xb2f325e2}


def test_generator_reproduces_the_reference_backend_hash_and_extends_it():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gen_backend_ph.py"), "--check-only", "--registry", REGISTRY], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert out.returncode == 0, out.stdout
    assert "7-backend hash reproduced: (backend >> 15) % 7 + 0" in out.stdout
    assert "8-backend hash" in out.stdout
    assert {n[len("CCV_NNC_BACKEND_"):]: v for n, v in json.load(open(REGISTRY))["backends"]} == REFERENCE_BACKENDS


def reference_cmd_inc(path):
    """The reference's ccv_nnc_cmd.inc in the shape its generator writes (the parts integration/patch_cmd_inc.py edits), rendered from the
    extracted tables: backend_init_map, the 7-slot _ccv_nnc_cmd_backend_ph, and _ccv_nnc_cmd_init() with every registration call, the
    GPU backends' under HAVE_CUDA."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_backend_ph as g
    t = json.load(open(REGISTRY))
    top, cases = t["backend_ph"]["top"], {int(i): tuple(p) for i, p in t["backend_ph"]["cases"].items()}
    params = [cases.get(i) for i in range(top[1])]
    by_slot = sorted(t["backends"], key=lambda nv: g.param_hash(nv[1], *cases[(nv[1] >> top[0]) % top[1]]))
    call = "\t_register_command_%s_backend_%s(&(init_map[%d].backends[%d]));\n"
    cpu = "".join(call % tuple(c) for c in t["calls"] if not c[1].startswith("CCV_NNC_BACKEND_GPU_"))
    gpu = "".join(call % tuple(c) for c in t["calls"] if c[1].startswith("CCV_NNC_BACKEND_GPU_"))
    text = ("static ccv_nnc_cmd_backend_init_t backend_init_map[] = {\n" + "".join('\t{.name = "%s", .backend = 0x%x},\n' % tuple(nv) for nv in by_slot) + "};\n\n"
            + g.c_switch("_ccv_nnc_cmd_backend_ph", "backend", (top[0], top[1], 0), params, False) + "\n"
            + "static inline void _ccv_nnc_cmd_init(void)\n{\n" + cpu + "#ifdef HAVE_CUDA\n" + gpu + "#endif\n}\n")
    open(path, "w").write(text)
    return text


def test_host_dispatch_goes_through_the_generated_tables():
    nnc.init()
    ok = nnc.lib().ccv_nnc_cmd_ok
    # every command the header lists is registered under GPU_SM100 and under no other backend id
    for name in dir(abi):
        if name.startswith("CCV_NNC_") and (name.endswith("_FORWARD") or name.endswith("_BACKWARD")) and isinstance(getattr(abi, name), int):
            cmd = getattr(abi, name)
            if ok(cmd, abi.CCV_NNC_BACKEND_GPU_SM100):
                for other in REFERENCE_BACKENDS.values():
                    assert ok(cmd, other) == 0, (name, hex(other))
    assert ok(abi.CCV_NNC_CONVOLUTION_FORWARD, abi.CCV_NNC_BACKEND_GPU_SM100) == 1
    assert ok(abi.CCV_NNC_CONVOLUTION_FORWARD, 0x12345678) == 0          # not a backend id
    assert ok(0x0badc0de, abi.CCV_NNC_BACKEND_GPU_SM100) == 0           # not a command id
    # generated fragments are committed next to the integration notes
    for f in ("ccv_nnc_backend.h", "ccv_nnc_cmd_backend.inc", "ccv_nnc_cmd_sm100_init.inc"):
        text = open(os.path.join(ROOT, "integration", f)).read()
        assert "CCV_NNC_BACKEND_GPU_SM100" in text
    assert "CCV_NNC_BACKEND_COUNT = 8" in open(os.path.join(ROOT, "integration", "ccv_nnc_backend.h")).read()


def test_patched_cmd_inc_reslots_every_registration_call(tmp_path):
    """integration/patch_cmd_inc.py (what build-cmd.rb would regenerate for an 8th backend): every `_register_command_X_backend_Y` call of the
    reference's generated file lands on the slot the 8-slot hash gives Y, the command slot is untouched, backend_init_map is ordered by
    slot (lib/nnc/ccv_nnc_cmd.c:61-66 requires backend_init_map[ph(b)].backend == b) and every SM100 registration of the header is present."""
    import re
    src, dst = str(tmp_path / "reference_ccv_nnc_cmd.inc"), str(tmp_path / "ccv_nnc_cmd.inc")
    ref = reference_cmd_inc(src)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "integration", "patch_cmd_inc.py"), src, dst], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    assert out.returncode == 0, out.stdout
    text = open(dst).read()
    backends = re.findall(r'\{\.name = "(CCV_NNC_BACKEND_[A-Z0-9_]+)", \.backend = (0x[0-9a-f]+)\}', text)
    assert len(backends) == 8

    def ph8(b):  # integration/ccv_nnc_cmd_backend.inc
        return ((b >> 2) % 8) if (b % 2 == 0) else ((b >> 9) % 8)
    for slot, (name, ident) in enumerate(backends):
        assert ph8(int(ident, 16)) == slot, (name, slot)
    slot_of = {name: i for i, (name, _) in enumerate(backends)}
    call = re.compile(r"_register_command_(CCV_NNC_[A-Z0-9_]+?)_backend_(CCV_NNC_BACKEND_[A-Z0-9_]+)\(&\(init_map\[(\d+)\]\.backends\[(\d+)\]\)\);")
    new_calls, old_calls = call.findall(text), call.findall(ref)
    n_sm100 = len(re.findall(r"X\(CCV_NNC_[A-Z0-9_]+\)", open(os.path.join(ROOT, "include", "ccv_nnc_sm100.h")).read()))  # CCV_NNC_SM100_COMMANDS
    assert len(old_calls) == 334 and len(new_calls) == 334 + n_sm100 and n_sm100 >= 94
    for cmd, backend, i, j in new_calls:
        assert int(j) == slot_of[backend], (cmd, backend, j)
    # the command slot of every pre-existing call is the reference's
    assert sorted((c, b, i) for c, b, i, _ in old_calls) == sorted((c, b, i) for c, b, i, _ in new_calls if b != "CCV_NNC_BACKEND_GPU_SM100")
    # an SM100 call uses the command slot its command already has
    cmd_slot = {c: i for c, _, i, _ in old_calls}
    sm100 = [(c, i) for c, b, i, _ in new_calls if b == "CCV_NNC_BACKEND_GPU_SM100"]
    assert len(sm100) == n_sm100 and all(cmd_slot[c] == i for c, i in sm100)
