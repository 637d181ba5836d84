"""Re-host the reference for the `--impl reference` arm of bench.py.

The reference (hangxu0304/DeepReduce) is not pip-installable: it has no
setup.py/pyproject, and its dependencies (grace_dl, cupy, pybloomfilter, mmh3,
dahuffman) plus its precomputed hash-table file are not available offline.  So the
install is a byte-identical copy of its `pytorch/deepreduce.py` into the git-ignored
`oracle/_ref/`; the missing third-party modules are provided by the minimal shims in
`baseline/shims/` (GRACE contract per SURVEY Appendix A; cupy packbits/unpackbits via
torch ops).  Nothing of deepreduce_b200 is on that path.

The source is a checkout of the reference: the directory named by the environment
variable ``DEEPREDUCE_REFERENCE``, else ``reference_path`` of BASELINE.json (relative
to the repository root: a checkout named ``reference`` next to this repository).
Without one the install is skipped, ``build()`` says so, and the reference arm reports
itself unavailable.
"""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
DST_DIR = os.path.join(HERE, "_ref", "deepreduce_ref")
DST = os.path.join(DST_DIR, "deepreduce.py")


def reference_root():
    root = os.environ.get("DEEPREDUCE_REFERENCE")
    if not root:
        with open(os.path.join(REPO, "BASELINE.json")) as f:
            root = json.load(f)["reference_path"]
    return os.path.normpath(os.path.join(REPO, root))      # an absolute path stays as it is


def install(verbose=True):
    if os.path.exists(DST):
        return DST
    src = os.path.join(reference_root(), "pytorch", "deepreduce.py")
    if not os.path.exists(src):
        if verbose:
            print(f"[oracle] no reference checkout at {os.path.dirname(os.path.dirname(src))} (set DEEPREDUCE_REFERENCE): "
                  "`bench.py --impl reference` will report itself unavailable")
        return None
    os.makedirs(DST_DIR, exist_ok=True)
    shutil.copyfile(src, DST)
    open(os.path.join(DST_DIR, "__init__.py"), "w").close()
    digest = hashlib.sha256(open(DST, "rb").read()).hexdigest()
    with open(os.path.join(DST_DIR, "SOURCE.txt"), "w") as f:
        f.write(f"copied unmodified from {src}\nsha256 {digest}\n")
    if verbose:
        print(f"[oracle] installed reference -> {DST} (sha256 {digest[:16]}…)")
    return DST


if __name__ == "__main__":
    sys.exit(0 if install() else 1)
