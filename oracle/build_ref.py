"""oracle/_ref recipe: the UNMODIFIED reference, byte-compiled where it lies.  TEST INFRASTRUCTURE.

    python oracle/build_ref.py [--reference DIR]

The reference is Python: "building" it means `py_compile` of the handful of files on the hot path,
straight from the sources of a reference checkout ($DPM_REFERENCE, default a `reference` directory next to this
repository or next to one of its parent directories)
into oracle/_ref/*.pyc (git-ignored; the bytecode may be copied to a GPU machine like our own .so, the sources never
enter the repo). A machine with the same CPython (same magic number) imports the .pyc files unchanged -- that is
how `-m gpu` tests, smoke() and `bench.py --impl reference` execute the real reference on the box
(`cpu_baseline.kind = "reference"`) where no reference checkout exists.

Only tests/, __graft_entry__ and bench.py's reference/cpu_baseline legs load these (oracle/ref_loader.py);
the product package never does.
"""
import argparse
import json
import os
import py_compile
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def _find_reference():
    """$DPM_REFERENCE, else a `reference` checkout next to this repository or next to any directory above it (a
    clean checkout may sit a few levels below the directory that holds the reference)."""
    if os.environ.get("DPM_REFERENCE"):
        return os.environ["DPM_REFERENCE"]
    repo = os.path.dirname(HERE)
    d = os.path.dirname(repo)
    while True:
        cand = os.path.join(d, "reference")
        if os.path.isfile(os.path.join(cand, "dpm_solver_pytorch.py")):
            return cand
        up = os.path.dirname(d)
        if up == d:
            return os.path.join(os.path.dirname(repo), "reference")
        d = up


DEFAULT_REFERENCE = _find_reference()
OUT = os.path.join(HERE, "_ref")

# logical name -> path under the reference tree
FILES = {
    # the solver itself (SURVEY 8a: every row cites this file)
    "dpm_solver_pytorch": "dpm_solver_pytorch.py",
    # Stable-Diffusion adapter + its vendored (older) solver copy (SURVEY 8b "who calls it")
    "sd_sampler": "examples/stable-diffusion/ldm/models/diffusion/dpm_solver/sampler.py",
    "sd_dpm_solver": "examples/stable-diffusion/ldm/models/diffusion/dpm_solver/dpm_solver.py",
    # score_sde glue (get_dpm_solver_sampler)
    "score_sde_sampling": "examples/score_sde_pytorch/sampling.py",
    # guided-diffusion runner (Diffusion.sample_image: classifier guidance + dynamic thresholding) and
    # the solver copy it imports
    "guided_runner": "examples/ddpm_and_guided-diffusion/runners/diffusion.py",
    "guided_sampler": "examples/ddpm_and_guided-diffusion/dpm_solver/sampler.py",
}


def build_ref(reference=DEFAULT_REFERENCE, quiet=False):
    """Byte-compile FILES into oracle/_ref/. Returns the manifest, or None when the reference tree is
    absent (prebuilt files, if any, are used as they are)."""
    if not os.path.isfile(os.path.join(reference, FILES["dpm_solver_pytorch"])):
        return None
    os.makedirs(OUT, exist_ok=True)
    manifest = {"python": sys.version.split()[0], "files": {}}
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", SyntaxWarning)      # the reference's docstrings contain "\h" etc.
        for name, rel in FILES.items():
            src = os.path.join(reference, rel)
            dst = os.path.join(OUT, name + ".pyc")
            py_compile.compile(src, cfile=dst, dfile=rel, doraise=True)
            manifest["files"][name] = {"source": rel, "bytes": os.path.getsize(src)}
    with open(os.path.join(OUT, "MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1)
    if not quiet:
        print("oracle/_ref: compiled", ", ".join(FILES))
    return manifest


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=DEFAULT_REFERENCE)
    a = ap.parse_args()
    if build_ref(a.reference) is None:
        print("reference tree not found at", a.reference, "- keeping the prebuilt oracle/_ref", file=sys.stderr)
