"""A/B builds of the engine with compile-time switches:

    python profiles/micro/build_variant.py TAG -DCWTB_UNROLL_A=8 [...]

writes pycwt_b200/variants/libcwtb200_TAG.so (git-ignored like every built library; it travels to
the GPU box with the snapshot).  Load it with `_engine.Engine(0, lib_path=...)`; the scripts under
profiles/micro/ take library paths as arguments.  The product only ever loads the in-tree
pycwt_b200/libcwtb200.so."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from pycwt_b200 import build as b   # noqa: E402


def main():
    tag, flags = sys.argv[1], sys.argv[2:]
    out_dir = os.path.join(ROOT, "pycwt_b200", "variants")
    os.makedirs(out_dir, exist_ok=True)
    lib = os.path.join(out_dir, "libcwtb200_%s.so" % tag)
    subprocess.check_call([b.NVCC] + b.FLAGS + ["-w"] + flags + [b.SRC, "-o", lib])
    print(lib)


if __name__ == "__main__":
    main()
