#!/usr/bin/env python
"""Vendor the reference files the hot path (and the stage-2 transformer, SURVEY.md 8f-3) lives in into oracle/_ref/
(git-ignored, like a built .so).

    python oracle/build_ref.py            # REFERENCE_ROOT overrides the checkout location; no-op where none is found

The files are copied byte for byte -- enhancing/modules/stage1/layers.py and quantizers.py import only torch / numpy /
einops -- so that `bench.py --impl reference`, `cpu_baseline` and `gpu_eager_baseline` time the REFERENCE's own
nn.Modules (kind "reference") instead of the oracle port, and so that oracle/gen_golden_ref_modules.py can record their
outputs as golden vectors.  Nothing under oracle/_ref is ever committed or imported by the product package."""
import hashlib
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.environ.get("REFERENCE_ROOT", "/root/reference")
FILES = ("enhancing/modules/stage1/layers.py", "enhancing/modules/stage1/quantizers.py")
# copied under another file name (stage 1 also has a layers.py); imports `omegaconf` for a type annotation only -- tests stub it
RENAMED = {"enhancing/modules/stage2/layers.py": "stage2_layers.py"}


def main() -> int:
    if not all(os.path.exists(os.path.join(SRC, f)) for f in FILES):
        print(f"oracle/build_ref.py: {SRC} not present -- keeping whatever oracle/_ref already holds")
        return 0
    dst = os.path.join(HERE, "_ref", "enhancing_ref")
    os.makedirs(dst, exist_ok=True)
    lines = []
    for f in FILES + tuple(RENAMED):
        if not os.path.exists(os.path.join(SRC, f)):
            continue
        out = os.path.join(dst, RENAMED.get(f, os.path.basename(f)))
        shutil.copyfile(os.path.join(SRC, f), out)
        lines.append(f"{hashlib.sha256(open(out, 'rb').read()).hexdigest()}  {f}")
    with open(os.path.join(dst, "SOURCE.txt"), "w") as fh:
        fh.write("unmodified copies of (sha256, path under the reference repository):\n" + "\n".join(lines) + "\n")
    print("oracle/_ref/enhancing_ref: " + ", ".join(sorted(x for x in os.listdir(dst) if x.endswith(".py"))))
    return 0


if __name__ == "__main__":
    sys.exit(main())
