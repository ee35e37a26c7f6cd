"""Writes tests/golden/kg_start_parent_counters.json: the q-KG counters (posterior evaluations, accepted steps, POINT
rounds, LINE batches, samples) of every case of tests/test_gpu_kg_start.py, as computed by a library that starts each
sample's inner descent with a POINT round (the commit before the start-point table).  Needs a GPU; the library is the
one CMOE_B200_LIB names.

    CMOE_B200_LIB=/path/to/parent/libcornell_moe_b200.so python tests/golden/make_kg_start_counters.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from cornell_moe_b200 import capi  # noqa: E402
from test_gpu_kg_start import CASES, GOLDEN, run_case  # noqa: E402


def main():
    assert capi.device_count() > 0, "no CUDA device"
    out = {name: run_case(capi, name)["stats"] for name in sorted(CASES)}
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
