"""Writes tests/golden/sm100_registry.json: the registry entry each GPU_SM100 registration function fills (formats, datatypes, memory,
algorithm count, which of exec / autotune / aux are set), the commands that share one exec function, and the commands whose exec only
returns CCV_NNC_EXEC_INVALID (the backward of SGD, ADAM, ADAMW, LAMB, RMSPROP, ARGMAX, ARGMIN, REDUCE_ISNAN and HISTOGRAM, which have
no gradient).  tests/test_registry_cpu.py compares the built library against it.

  python tests/golden/make_registry_golden.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.test_registry_cpu import SM100_REGISTRY, registry_snapshot  # noqa: E402

INVALID_EXEC = ["CCV_NNC_%s_BACKWARD" % c for c in ("ADAM", "ADAMW", "ARGMAX", "ARGMIN", "HISTOGRAM", "LAMB", "REDUCE_ISNAN", "RMSPROP", "SGD")]

if __name__ == "__main__":
    snap = registry_snapshot()
    snap["invalid_exec"] = INVALID_EXEC
    with open(SM100_REGISTRY, "w") as f:
        json.dump(snap, f, indent=1, sort_keys=True)
        f.write("\n")
