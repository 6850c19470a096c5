#!/usr/bin/env python
"""Merge the reports of integration/run_reference_tests.py (a full run, then retries of what failed after fixes) into one table of the
reference's own test cases on the drop-in build: <name>.json and <name>.md.

  python tools/dropin_table.py <name> run_full.json [retry1.json ...]"""
import json
import sys


def main(out, paths):
    merged = {}
    for path in paths:
        rep = json.load(open(path))["programs"]
        for prog, r in rep.items():
            m = merged.setdefault(prog, {})
            for k in r.get("passed", []):
                m[k] = ("PASS", "")
            for k in r.get("skipped", []):
                m[k] = ("SKIP", "")
            for k, v in r.get("fail_detail", {}).items():
                m[k] = ("FAIL", v)
            for k in r.get("failed", []):
                m.setdefault(k, ("FAIL", ""))
            for k, v in r.get("crashed", {}).items():
                m[k] = ("CRASH", v)
    total = {}
    lines = ["| program (test/{int,unit}/nnc/*.tests.c of the reference, unmodified) | PASS | SKIP | FAIL | CRASH |", "|---|---|---|---|---|"]
    for prog in sorted(merged):
        t = {s: sum(1 for v in merged[prog].values() if v[0] == s) for s in ("PASS", "SKIP", "FAIL", "CRASH")}
        for s, n in t.items():
            total[s] = total.get(s, 0) + n
        lines.append("| %s | %d | %d | %d | %d |" % (prog, t["PASS"], t["SKIP"], t["FAIL"], t["CRASH"]))
    lines.append("| **total** | **%d** | %d | %d | %d |" % (total.get("PASS", 0), total.get("SKIP", 0), total.get("FAIL", 0), total.get("CRASH", 0)))
    lines += ["", "Cases that do not pass:", ""]
    for prog in sorted(merged):
        for k, (s, d) in sorted(merged[prog].items()):
            if s in ("FAIL", "CRASH"):
                d = d.replace("\x1b[0;31m", "").replace("\x1b[0;0m", "").replace("|", "/")
                lines.append("* `%s` -- **%s** %s: %s" % (prog, s, k, d[-330:]))
    json.dump({"total": total, "programs": {p: {k: {"status": v[0], "detail": v[1]} for k, v in sorted(c.items())} for p, c in sorted(merged.items())}}, open(out + ".json", "w"), indent=1)
    open(out + ".md", "w").write("\n".join(lines) + "\n")
    print("\n".join(lines[:len(merged) + 3]))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2:])
