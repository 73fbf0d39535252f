"""Recipe for ``oracle/_ref`` (git-ignored output, test infrastructure): a byte-identical copy of exactly those files of the
reference tree that ``oracle/ref_loader.py`` imports for the hot path -- plain Python modules of
``/root/reference/src/schnetpack`` ({properties, utils, nn, representation, atomistic/{atomwise,response,distances},
transform/{base,atomistic,casting,neighborlist}, model/base}) -- plus the two small files of the reference's
``tests/testdata`` the parity tests use (``md_ethanol.model`` = the shipped trained PaiNN, ``md_ethanol.xyz``).

    python oracle/make_ref.py          # build container only (needs /root/reference); idempotent

``/root/reference`` does not exist on the GPU box, ``oracle/_ref`` travels there with the snapshot (it is git-ignored but not
gpurun-ignored), so the ``-m gpu`` tests can hold the CUDA path against the UNMODIFIED reference modules running on the same
GPU (``tests/test_reference_live.py``), and ``bench.py --impl reference`` / ``cpu_baseline`` time the reference itself
(``kind: "reference"``) instead of the oracle port.  Nothing is ever written to the reference tree, and no reference source
enters the git history.
"""
import hashlib
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
REF_ROOT = "/root/reference"
OUT = os.path.join(HERE, "_ref")
TESTDATA = ("md_ethanol.model", "md_ethanol.xyz")


def main() -> int:
    src_pkg = os.path.join(REF_ROOT, "src", "schnetpack")
    if not os.path.isdir(src_pkg):
        print("make_ref: /root/reference not present -- keeping the existing oracle/_ref (if any)")
        return 0
    from oracle import ref_loader as rl

    if rl.SOURCE != "tree":
        raise RuntimeError("ref_loader did not resolve to the reference tree")
    files = rl.loaded_files()
    # packages imported through stub parents have no __init__ of their own in sys.modules: the loader never needs one
    manifest = []
    for f in files:
        rel = os.path.relpath(f, src_pkg)
        dst = os.path.join(OUT, "schnetpack", rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(f, dst)
        manifest.append((os.path.join("schnetpack", rel), hashlib.sha256(open(f, "rb").read()).hexdigest()))
    os.makedirs(os.path.join(OUT, "testdata"), exist_ok=True)
    for name in TESTDATA:
        f = os.path.join(REF_ROOT, "tests", "testdata", name)
        shutil.copyfile(f, os.path.join(OUT, "testdata", name))
        manifest.append((os.path.join("testdata", name), hashlib.sha256(open(f, "rb").read()).hexdigest()))
    with open(os.path.join(OUT, "MANIFEST.sha256"), "w") as fh:
        for rel, h in sorted(manifest):
            fh.write(f"{h}  {rel}\n")
    print(f"make_ref: {len(manifest)} files -> {OUT}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
