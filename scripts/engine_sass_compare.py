"""Compare the SASS of the fused engine's existing kernel variants between a base commit and the working tree.

    python scripts/engine_sass_compare.py <base-commit>

Compiles ``ops/csrc/engine.cu`` of both trees for sm_90a with the flags of ``ops/build.py`` (no GPU needed), dumps
each cubin with ``cuobjdump -sass`` and compares, per ``dr_engine_kernel<blocks, full, bf16>`` instantiation of the
base, its instructions with the working tree's instantiation of the same first three template arguments, after the
function names are stripped.  Variants the base does not have (e.g. ``<.., .., .., true>``) are listed, not compared.
Exit code 0 when every base variant is byte-identical.
"""
from __future__ import annotations

import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = "deepreduce_b200/ops/csrc"
sys.path.insert(0, os.path.join(ROOT, "deepreduce_b200", "ops"))
from build import NVCC_FLAGS  # noqa: E402

CUBIN_FLAGS = [f for f in NVCC_FLAGS if f not in ("-Xcompiler", "-fPIC", "-Xptxas", "-v")]


def tool(name: str) -> str:
    return shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)


def export_base(rev: str, dst: str) -> None:
    files = subprocess.run(["git", "-C", ROOT, "ls-tree", "--name-only", f"{rev}:{CSRC}"], check=True,
                           capture_output=True, text=True).stdout.split()
    for f in files:
        if f.endswith((".cu", ".cuh", ".h")):
            blob = subprocess.run(["git", "-C", ROOT, "show", f"{rev}:{CSRC}/{f}"], check=True, capture_output=True).stdout
            with open(os.path.join(dst, f), "wb") as fh:
                fh.write(blob)


def kernels(src_dir: str, work: str, tag: str) -> dict:
    cubin = os.path.join(work, f"{tag}.cubin")
    subprocess.run([tool("nvcc")] + CUBIN_FLAGS + ["-I", src_dir, "-cubin", os.path.join(src_dir, "engine.cu"),
                                                   "-o", cubin], check=True)
    sass = subprocess.run([tool("cuobjdump"), "-sass", cubin], check=True, capture_output=True, text=True).stdout
    out = {}
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name, code = body.split("\n", 1)
        name = name.strip()
        if "dr_engine_kernel" not in name:
            continue
        pretty = subprocess.run([tool("cu++filt"), name], check=True, capture_output=True, text=True).stdout.strip()
        args = re.search(r"dr_engine_kernel<([^>]*)>", pretty).group(1).split(", ")
        # template arguments of a kernel in an anonymous namespace demangle as (int)2 / (bool)0
        args = [{"(bool)0": "false", "(bool)1": "true"}.get(a, re.sub(r"^\(int\)", "", a)) for a in args]
        # the instruction lines only: the section trailer that follows the last function is not code
        lines = [l.rstrip() for l in code.split("\n") if re.match(r"\s+/\*[0-9a-f]{4}\*/", l)
                 or re.match(r"\s+/\* 0x[0-9a-f]{16} \*/", l)]
        out[tuple(args)] = "\n".join(lines)
    return out


def main() -> int:
    if len(sys.argv) != 2:
        print(__doc__)
        return 2
    rev = sys.argv[1]
    with tempfile.TemporaryDirectory() as work:
        base_dir = os.path.join(work, "base")
        os.makedirs(base_dir)
        export_base(rev, base_dir)
        base = kernels(base_dir, work, "base")
        head = kernels(os.path.join(ROOT, CSRC), work, "head")
    ok = True
    for args, code in sorted(base.items()):
        n = len(args)                # 3 or 4 template arguments, depending on the base
        match = [c for a, c in head.items() if a[:n] == args and all(x == "false" for x in a[n:])]
        same = bool(match) and match[0] == code
        ok &= same
        print(f"dr_engine_kernel<{', '.join(args)}>: {code.count(chr(10)) + 1} lines, "
              f"{'identical' if same else 'DIFFERENT' if match else 'MISSING in the working tree'}")
    n = len(next(iter(base))) if base else 3
    for args in sorted(a for a in head if a[:n] not in base or any(x != "false" for x in a[n:])):
        print(f"dr_engine_kernel<{', '.join(args)}>: new variant ({head[args].count(chr(10)) + 1} lines)")
    print("all base variants identical" if ok else "SASS differs")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
