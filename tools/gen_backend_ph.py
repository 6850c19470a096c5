#!/usr/bin/env python
"""Registry plumbing for an 8th backend (SURVEY.md 8b, VERDICT r01 item 7): re-derives the perfect hashes of the reference's
generated lib/nnc/cmd/ccv_nnc_cmd.inc and extends the backend side to CCV_NNC_BACKEND_GPU_SM100.

The reference generates `_ccv_nnc_cmd_ph` / `_ccv_nnc_cmd_backend_ph` with a small hash-displace-compress search written in
Ruby (lib/nnc/cmd/build-cmd.rb:303-386; Ruby is not in this image).  This tool states the same search in Python:

  h(key; idx, n, off) = (key >> idx) % n + off            one family of hash functions over the 32-bit SHA-256 prefix ids
  top level:  smallest bucket count i (then smallest bit offset k) for which every bucket b -- visited largest first -- finds
              parameters (idx_b, n_b, off_b), tried in the order idx, n >= |b|, off, that place its keys on distinct free slots.

and checks itself against the reference before emitting anything:
  * run on the reference's 7 backends it must reproduce the committed `_ccv_nnc_cmd_backend_ph`   ((backend >> 15) % 7 + 0),
  * the committed `_ccv_nnc_cmd_ph` must be a perfect hash of the reference's command ids onto 0 .. 2 * 69 (evaluated from the
    constants parsed out of the .inc itself -- the command table is untouched by a new backend).
Then it emits, for the 8-backend set, the files a ccv maintainer would regenerate (integration/):
  ccv_nnc_backend.h            the enum with CCV_NNC_BACKEND_GPU_SM100 = 0xdbfb784c and CCV_NNC_BACKEND_COUNT = 8
  ccv_nnc_cmd_backend.inc      backend_init_map[8] + the 8-slot _ccv_nnc_cmd_backend_ph
  ccv_nnc_cmd_sm100_init.inc   the prototype and the `_register_command_..._backend_CCV_NNC_BACKEND_GPU_SM100(...)` call per command
and ccv_b200/csrc/nnc_registry_generated.inc, which the stand-alone host (nnc_host.cu) compiles: the same two hash functions,
so that its init_map[cmd].backends[8] / ccv_nnc_cmd_find_backend walk the slots exactly as lib/nnc/ccv_nnc_cmd.c:307-328 does.

  python tools/gen_backend_ph.py [--registry FILE] [--check-only]

FILE is the reference's lib/nnc/cmd/ccv_nnc_cmd.inc, or (the default) tests/golden/reference_cmd_registry.json: the same tables
extracted from it by tests/golden/make_golden.py, so that the checks run without the reference tree.
"""
import argparse
import hashlib
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_BACKEND = "CCV_NNC_BACKEND_GPU_SM100"


def sha_id(name):
    return int(hashlib.sha256(name.encode()).hexdigest()[:8], 16)  # build-cmd.rb:386


def param_hash(val, idx, n, off):
    return (val >> idx) % n + off


def perfect_hashing(keys, hashval):
    """keys: ordered list of names; hashval: name -> 32-bit value.  Returns (top_level, bucket_params, mapping)."""
    count = len(keys)
    for i in range(1, count + 1):
        for k in range(0, 31):
            buckets = [[] for _ in range(i)]
            for key in keys:
                buckets[param_hash(hashval[key], k, i, 0)].append(key)
            order = sorted((b for b in enumerate(buckets) if b[1]), key=lambda b: len(b[1]), reverse=True)
            taken = [False] * count
            params, mapping, ok = [None] * i, {}, True
            for bidx, bkeys in order:
                found = None
                for j in range(0, 31):
                    for x in range(len(bkeys), count + 1):
                        vals = [param_hash(hashval[key], j, x, 0) for key in bkeys]
                        if len(set(vals)) != len(vals):
                            continue
                        for y in range(0, count - x + 1):
                            if not any(taken[v + y] for v in vals):
                                found = (j, x, y)
                                break
                        if found:
                            break
                    if found:
                        break
                if not found:
                    ok = False
                    break
                for key in bkeys:
                    v = param_hash(hashval[key], *found)
                    mapping[key] = v
                    taken[v] = True
                params[bidx] = found
            if ok:
                return (k, i, 0), params, mapping
    raise RuntimeError("no perfect hash found")


def parse_inc(path):
    """(commands, backends, command-hash top level, its buckets, backend-hash top level, its buckets) of a generated ccv_nnc_cmd.inc, or
    of the JSON fixture holding the same tables."""
    if path.endswith(".json"):
        t = json.load(open(path))
        cases = {int(i): tuple(p) for i, p in t["cmd_ph"]["cases"].items()}
        bcases = {int(i): tuple(p) for i, p in t["backend_ph"]["cases"].items()}
        return [tuple(c) for c in t["commands"]], [tuple(b) for b in t["backends"]], tuple(t["cmd_ph"]["top"]), cases, tuple(t["backend_ph"]["top"]), bcases
    text = open(path).read()
    cmds = re.findall(r'\{\.name = "(CCV_NNC_[A-Z0-9_]+)", \.cmd = (0x[0-9a-f]+)\}', text)
    backends = re.findall(r'\{\.name = "(CCV_NNC_BACKEND_[A-Z0-9_]+)", \.backend = (0x[0-9a-f]+)\}', text)
    m = re.search(r"static inline int _ccv_nnc_cmd_ph\(const uint32_t cmd\)\s*\{\s*switch \(\(cmd >> (\d+)\) % (\d+)\)(.*?)\n\}\n", text, re.S)
    top = (int(m.group(1)), int(m.group(2)))
    cases = {}
    for cm in re.finditer(r"case (\d+):(?:\s*default:)?\s*return \(\(\(\(cmd >> (\d+)\) % (\d+)\) \+ (\d+)\) << 1\) \| \(cmd & 1\);", m.group(3)):
        cases[int(cm.group(1))] = (int(cm.group(2)), int(cm.group(3)), int(cm.group(4)))
    b = re.search(r"static inline int _ccv_nnc_cmd_backend_ph\(const uint32_t backend\)\s*\{\s*switch \(\(backend >> (\d+)\) % (\d+)\)(.*?)\n\}\n", text, re.S)
    btop = (int(b.group(1)), int(b.group(2)))
    bcases = {}
    for cm in re.finditer(r"case (\d+):(?:\s*default:)?\s*return \(\(backend >> (\d+)\) % (\d+)\) \+ (\d+);", b.group(3)):
        bcases[int(cm.group(1))] = (int(cm.group(2)), int(cm.group(3)), int(cm.group(4)))
    return [(n, int(v, 16)) for n, v in cmds], [(n, int(v, 16)) for n, v in backends], top, cases, btop, bcases


REGISTER_CALL = re.compile(r"_register_command_(CCV_NNC_[A-Z0-9_]+?)_backend_(CCV_NNC_BACKEND_[A-Z0-9_]+)\(&\(init_map\[(\d+)\]\.backends\[(\d+)\]\)\);")


def registration_calls(text):
    """(command, backend, command slot, backend slot) of every registration call in a generated ccv_nnc_cmd.inc."""
    return [(c, b, int(i), int(j)) for c, b, i, j in REGISTER_CALL.findall(text)]


def c_switch(fn, arg, top, params, pair):
    k, n, _ = top
    lines = ["static inline int %s(const uint32_t %s)" % (fn, arg), "{", "\tswitch ((%s >> %d) %% %d)" % (arg, k, n), "\t{"]
    for i, p in enumerate(params):
        if p is None:
            continue
        last = i == max(j for j, q in enumerate(params) if q is not None)
        lines.append("\t\tcase %d:" % i)
        if last:
            lines.append("\t\tdefault:")
        if pair:
            lines.append("\t\t\treturn ((((%s >> %d) %% %d) + %d) << 1) | (%s & 1);" % (arg, p[0], p[1], p[2], arg))
        else:
            lines.append("\t\t\treturn ((%s >> %d) %% %d) + %d;" % (arg, p[0], p[1], p[2]))
    lines += ["\t}", "}"]
    return "\n".join(lines) + "\n"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--registry", default=os.path.join(ROOT, "tests", "golden", "reference_cmd_registry.json"))
    ap.add_argument("--check-only", action="store_true")
    args = ap.parse_args()
    cmds, backends, top, cases, btop, bcases = parse_inc(args.registry)
    assert len(cmds) % 2 == 0 and all(sha_id(n[:-len("_FORWARD")]) & ~1 == v for n, v in cmds if n.endswith("_FORWARD")), "command ids are not SHA-256 prefixes"  # build-cmd.rb:292
    assert all(sha_id(n) == v for n, v in backends), "backend ids are not SHA-256 prefixes"

    # 1. the committed command hash is perfect over the committed command ids
    def ref_cmd_ph(cmd):
        j, x, y = cases[(cmd >> top[0]) % top[1]]
        return ((((cmd >> j) % x) + y) << 1) | (cmd & 1)
    slots = sorted(ref_cmd_ph(v) for _, v in cmds)
    assert slots == list(range(len(cmds))), "reference _ccv_nnc_cmd_ph is not a perfect hash?"

    # 2. this search reproduces the committed backend hash on the reference's own 7 backends
    names7 = [n for n, _ in backends]
    t7, p7, _ = perfect_hashing(names7, dict(backends))
    assert (t7[0], t7[1]) == btop and {i: p for i, p in enumerate(p7) if p is not None} == bcases, ("backend hash differs from the reference's", t7, p7, btop, bcases)
    # ... and the committed command hash too (keys = command names, value = id >> 1: build-cmd.rb:379).  The search visits buckets
    # largest first; Ruby's sort is unstable and the generator's input order (file-system order of the command sources) is not
    # recorded in the .inc, so equal-sized buckets may be visited in another order here: then the result is another, equally
    # valid, perfect hash -- the committed one stays authoritative (it is the one evaluated above and emitted below)
    fwd = [(n, v) for n, v in cmds if v & 1 == 0]
    tc, pc, mc = perfect_hashing([n for n, _ in fwd], dict((n, v >> 1) for n, v in fwd))
    assert sorted(mc.values()) == list(range(len(fwd)))
    same_cmd = (tc[1] == top[1] and tc[0] + 1 == top[0] and all(cases.get(i) == (p[0] + 1, p[1], p[2]) for i, p in enumerate(pc) if p is not None))
    print("7-backend hash reproduced: (backend >> %d) %% %d + %d; command hash over %d commands: top level (cmd >> %d) %% %d %s" % (
        p7[0][0], p7[0][1], p7[0][2], len(fwd), tc[0] + 1, tc[1], "reproduced bucket for bucket" if same_cmd else "found (same top level: %s; bucket parameters differ by tie-breaking)" % (tc[1] == top[1] and tc[0] + 1 == top[0])))

    # 3. the 8-backend set
    new_id = sha_id(NEW_BACKEND)
    assert new_id == 0xdbfb784c
    backends8 = backends + [(NEW_BACKEND, new_id)]
    t8, p8, map8 = perfect_hashing([n for n, _ in backends8], dict(backends8))
    assert sorted(map8.values()) == list(range(8))
    print("8-backend hash: top (backend >> %d) %% %d, buckets %s" % (t8[0], t8[1], [p for p in p8 if p is not None]))
    if args.check_only:
        return
    backend_ph = c_switch("_ccv_nnc_cmd_backend_ph", "backend", t8, p8, False)
    # backend_init_map is indexed by the hash (lib/nnc/ccv_nnc_cmd.c:61-66 checks backend_init_map[ph(b)].backend == b)
    ordered = sorted(backends8, key=lambda nv: map8[nv[0]])
    init_map = "static ccv_nnc_cmd_backend_init_t backend_init_map[] = {\n" + "".join('\t{.name = "%s", .backend = 0x%x},\n' % nv for nv in ordered) + "};\n"
    out = os.path.join(ROOT, "integration")
    os.makedirs(out, exist_ok=True)
    enum_lines = "".join("\t%s = 0x%x,\n" % nv for nv in sorted(backends8))
    open(os.path.join(out, "ccv_nnc_backend.h"), "w").write(
        "/* regenerated by tools/gen_backend_ph.py: lib/nnc/cmd/ccv_nnc_backend.h with the SM100 backend added */\n/**\n * @addtogroup available_backends Available Backends\n * @{\n */\nenum {\n\tCCV_NNC_NO_BACKEND = 0,\n"
        + enum_lines + "\tCCV_NNC_BACKEND_COUNT = 8,\n};\n/** @} */\n")
    open(os.path.join(out, "ccv_nnc_cmd_backend.inc"), "w").write(
        "/* regenerated by tools/gen_backend_ph.py: the two backend-side pieces of lib/nnc/cmd/ccv_nnc_cmd.inc (lines 142-190) for 8 backends */\n" + init_map + "\n" + backend_ph)
    header = open(os.path.join(ROOT, "include", "ccv_nnc_sm100.h")).read()
    # the first list, then the per-family lists that follow the declaration macro
    sm100_cmds = re.findall(r"X\((CCV_NNC_[A-Z0-9_]+)\)", header[header.index("#define CCV_NNC_SM100_COMMANDS(X)"):header.index("#define CCV_SM100_DECLARE_REGISTER")])
    sm100_cmds += re.findall(r"X\((CCV_NNC_[A-Z0-9_]+)\)", header[header.index("#define CCV_NNC_SM100_DETECTION_COMMANDS(X)"):header.index("CCV_NNC_SM100_DETECTION_COMMANDS(CCV_SM100_DECLARE_REGISTER)")])
    sm100_cmds += re.findall(r"X\((CCV_NNC_[A-Z0-9_]+)\)", header[header.index("#define CCV_NNC_SM100_OPTIMIZER_COMMANDS(X)"):header.index("CCV_NNC_SM100_OPTIMIZER_COMMANDS(CCV_SM100_DECLARE_REGISTER)")])
    sm100_cmds += re.findall(r"X\((CCV_NNC_[A-Z0-9_]+)\)", header[header.index("#define CCV_NNC_SM100_COMPRESSION_COMMANDS(X)"):header.index("CCV_NNC_SM100_COMPRESSION_COMMANDS(CCV_SM100_DECLARE_REGISTER)")])
    sm100_cmds += re.findall(r"X\((CCV_NNC_[A-Z0-9_]+)\)", header[header.index("#define CCV_NNC_SM100_STATISTICS_COMMANDS(X)"):header.index("CCV_NNC_SM100_STATISTICS_COMMANDS(CCV_SM100_DECLARE_REGISTER)")])
    ids = dict(cmds)
    lines = ["/* regenerated by tools/gen_backend_ph.py: what build-cmd.rb adds to ccv_nnc_cmd.inc for every (command, GPU_SM100) pair */"]
    for c in sm100_cmds:
        lines.append("void _register_command_%s_backend_%s(ccv_nnc_cmd_backend_registry_t* const registry);" % (c, NEW_BACKEND))
    lines.append("\nstatic inline void _ccv_nnc_cmd_init_sm100(void)\n{")
    for c in sm100_cmds:
        lines.append("\t_register_command_%s_backend_%s(&(init_map[%d].backends[%d]));" % (c, NEW_BACKEND, ref_cmd_ph(ids[c]), map8[NEW_BACKEND]))
    lines.append("}\n")
    open(os.path.join(out, "ccv_nnc_cmd_sm100_init.inc"), "w").write("\n".join(lines))
    # the stand-alone host's copy: command hash (the reference's, evaluated above as a perfect hash) + the 8-slot backend hash
    cmd_params = [None] * top[1]
    for i, p in cases.items():
        cmd_params[i] = p
    gen = ["/* GENERATED by tools/gen_backend_ph.py -- do not edit.  The perfect hashes the stand-alone host dispatches with: the command",
           " * hash of lib/nnc/cmd/ccv_nnc_cmd.inc (unchanged by a new backend; verified perfect over the reference's %d command ids) and the" % len(cmds),
           " * 8-slot backend hash found by the same hash-displace-compress search with CCV_NNC_BACKEND_GPU_SM100 added. */",
           "#define CCV_NNC_SM100_CMD_SLOTS %d" % len(cmds), "#define CCV_NNC_SM100_BACKEND_SLOTS 8", "",
           c_switch("_ccv_nnc_cmd_ph", "cmd", (top[0], top[1], 0), cmd_params, True),
           c_switch("_ccv_nnc_cmd_backend_ph", "backend", t8, p8, False),
           "static const struct { const char* name; uint32_t backend; } sm100_backend_init_map[CCV_NNC_SM100_BACKEND_SLOTS] = {"]
    gen += ['\t{ "%s", 0x%xu },' % nv for nv in ordered]
    gen += ["};", "static const struct { const char* name; uint32_t cmd; } sm100_cmd_init_map[CCV_NNC_SM100_CMD_SLOTS] = {"]
    by_slot = sorted(cmds, key=lambda nv: ref_cmd_ph(nv[1]))
    gen += ['\t{ "%s", 0x%xu },' % nv for nv in by_slot]
    gen += ["};", ""]
    open(os.path.join(ROOT, "ccv_b200", "csrc", "nnc_registry_generated.inc"), "w").write("\n".join(gen))
    print("wrote integration/{ccv_nnc_backend.h, ccv_nnc_cmd_backend.inc, ccv_nnc_cmd_sm100_init.inc} and ccv_b200/csrc/nnc_registry_generated.inc")


if __name__ == "__main__":
    main()
