"""Registers and stack bytes of every kernel of csrc/train.cu, as ptxas allocates them for sm_90a.

    python scripts/train_resources.py [--diff FILE]

Compiles train.cu with the package's own nvcc flags (torchkge_b200/_build.py) into a temporary directory,
reads `cuobjdump --dump-resource-usage` and prints one line per kernel instantiation, sorted:

    margin_step_ring_kernel<0, 1, 5, 0, 0> REG=96 STACK=192

(template arguments as integers: MODEL, BWD, MINB, SHARD, LOSS).  With --diff FILE the listing is compared
with one saved earlier and the exit code is 1 if any line differs.  The table of DESIGN.md section 4.4 is
this listing; a change to train.cu that moves a count shows up here before it reaches a GPU.  Needs nvcc,
cuobjdump and cu++filt (the CUDA toolkit); no GPU.
"""
import argparse
import difflib
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from torchkge_b200 import _build  # noqa: E402


def kernel_name(demangled):
    """`margin_step_fast_kernel<1, 0>` from cu++filt's `void kge::<unnamed>::margin_step_fast_kernel<(int)1,
    (bool)0>(kge::MarginStepParams, ...)`."""
    m = re.search(r"(\w+)(<[^<>]*>)?\(", demangled.replace("<unnamed>::", ""))
    args = re.sub(r"\(\w+\)", "", m.group(2) or "").replace("true", "1").replace("false", "0")
    return m.group(1) + args


def listing():
    nvcc = _build._nvcc()
    tool = lambda name: os.path.join(os.path.dirname(nvcc), name)  # noqa: E731
    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, "train.o")
        subprocess.check_call([nvcc] + _build.NVCC_FLAGS + ["-c", os.path.join(_build.CSRC, "train.cu"), "-o", obj])
        dump = subprocess.check_output([tool("cuobjdump"), "--dump-resource-usage", obj], text=True)
    found = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", dump)
    names = subprocess.check_output([tool("cu++filt")] + [f[0] for f in found], text=True).splitlines()
    return sorted("%s REG=%s STACK=%s" % (kernel_name(n), reg, stack) for n, (_, reg, stack) in zip(names, found))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--diff", metavar="FILE", default=None, help="a saved listing to compare with")
    args = ap.parse_args()
    now = listing()
    if args.diff is None:
        print("\n".join(now))
        return 0
    with open(args.diff) as f:
        saved = f.read().split("\n")
    saved = [s for s in saved if s.strip()]
    delta = list(difflib.unified_diff(saved, now, args.diff, "this tree", lineterm="", n=0))
    print("\n".join(delta) if delta else "no difference: %d kernels" % len(now))
    return 1 if delta else 0


if __name__ == "__main__":
    sys.exit(main())
