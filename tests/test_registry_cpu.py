"""The registry plumbing of an 8th backend (SURVEY.md 8b): tools/gen_backend_ph.py re-derives the reference's perfect hashes
(lib/nnc/cmd/build-cmd.rb:303-386, lib/nnc/cmd/ccv_nnc_cmd.inc:152-190) and the stand-alone host dispatches through
init_map[_ccv_nnc_cmd_ph(cmd)].backends[_ccv_nnc_cmd_backend_ph(backend)] exactly as lib/nnc/ccv_nnc_cmd.c does."""
import ctypes as C
import json
import os
import re
import subprocess
import sys

import pytest

from ccv_b200 import abi, nnc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the reference's generated registry tables (lib/nnc/cmd/ccv_nnc_cmd.inc), extracted by tests/golden/make_golden.py
REGISTRY = os.path.join(ROOT, "tests", "golden", "reference_cmd_registry.json")
# what every GPU_SM100 registration function writes, recorded by tests/golden/make_registry_golden.py
SM100_REGISTRY = os.path.join(ROOT, "tests", "golden", "sm100_registry.json")
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


class BackendRegistry(C.Structure):  # ccv_nnc_cmd_backend_registry_t
    _fields_ = [("tensor_formats", C.c_int), ("tensor_datatypes", C.c_int), ("tensor_memory", C.c_int), ("algorithms", C.c_int),
                ("exec", C.c_void_p), ("autotune", C.c_void_p), ("aux", C.c_void_p)]


def registry_snapshot():
    """Calls the registration function of every command include/ccv_nnc_sm100.h lists (no device needed: it only fills a record) and
    returns what each one wrote, plus the commands that share one exec function.  The grouping does not depend on addresses, so it
    tells a registration pointed at another command's exec apart from the same table."""
    lib = nnc.lib()
    cmds = re.findall(r"X\((CCV_NNC_[A-Z0-9_]+)\)", open(os.path.join(ROOT, "include", "ccv_nnc_sm100.h")).read())
    entries, by_exec = {}, {}
    for cmd in cmds:
        r = BackendRegistry()
        C.memset(C.byref(r), 0xa5, C.sizeof(r))
        getattr(lib, "_register_command_%s_backend_CCV_NNC_BACKEND_GPU_SM100" % cmd)(C.byref(r))
        entries[cmd] = {"tensor_formats": r.tensor_formats, "tensor_datatypes": r.tensor_datatypes, "tensor_memory": r.tensor_memory,
                        "algorithms": r.algorithms, "exec": bool(r.exec), "autotune": bool(r.autotune), "aux": bool(r.aux)}
        by_exec.setdefault(r.exec, []).append(cmd)
    return {"commands": entries, "exec_groups": sorted(sorted(g) for g in by_exec.values() if len(g) > 1)}


def test_every_sm100_registration_fills_the_recorded_entry():
    want = json.load(open(SM100_REGISTRY))
    got = registry_snapshot()
    assert len(got["commands"]) == len(want["commands"]) == 132
    for cmd, entry in want["commands"].items():
        assert got["commands"].get(cmd) == entry, cmd
    # The commands without a gradient register an exec that only returns CCV_NNC_EXEC_INVALID; whether they share one such function
    # or each family has its own is not part of the table.  Every other command keeps its exec grouping.
    invalid = set(want["invalid_exec"])

    def split(groups, singles):
        merged = [g for g in groups if invalid & set(g)] + [[c] for c in singles if c in invalid]
        return sorted(c for g in merged for c in g), [g for g in groups if not invalid & set(g)]
    singles = set(got["commands"]) - {c for g in got["exec_groups"] for c in g}
    got_invalid, got_groups = split(got["exec_groups"], singles)
    assert got_invalid == sorted(invalid)
    assert got_groups == [g for g in want["exec_groups"] if not invalid & set(g)]
