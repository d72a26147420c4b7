"""Writes tests/golden_buildlib/buildlib.json: for every case of tests/buildlib_cases.py, the exit status of the reference
`megahit_core buildlib` (oracle/_ref/megahit_core_ref) and the sha256 of the P.bin / P.lib_info it wrote.

    python scripts/gen_golden_buildlib.py
"""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import buildlib_cases as BC  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")


def run_reference(libs, exe=REF):
    with tempfile.TemporaryDirectory() as d:
        lib = BC.write_lib(d, libs)
        r = subprocess.run([exe, "buildlib", lib, os.path.join(d, "out")], capture_output=True)
        if r.returncode != 0:
            return {"rc": r.returncode}
        return {"rc": 0, **BC.digests(os.path.join(d, "out"))}


def main():
    if not os.access(REF, os.X_OK):
        sys.exit(f"{REF} is missing: build it with `make -C oracle ref`")
    out = {name: run_reference(libs) for name, libs in sorted(BC.all_cases().items())}
    path = os.path.join(ROOT, "tests", "golden_buildlib", "buildlib.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{len(out)} cases -> {path}")


if __name__ == "__main__":
    main()
