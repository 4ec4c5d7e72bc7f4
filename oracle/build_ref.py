"""Bundle the UNMODIFIED reference into oracle/_ref/gligen_reference.zip  (test infrastructure, not product code).

    python oracle/build_ref.py            # authoring container only: reads /root/reference, writes oracle/_ref/

The reference (gligen/GLIGEN) is a pure-Python script tree without setup.py / pyproject.toml, so there is nothing
to compile or pip-install; the equivalent of "building the reference into oracle/_ref" is an import-able archive of
its modules, byte for byte as they lie under /root/reference (python imports straight from a .zip).  The archive is
git-ignored (it never enters history); copied with the working tree to a GPU machine, where /root/reference does
not exist.  Users (all of them checkers, never the product path):

  * bench.py --impl reference : times the reference's own PLMSSampler + UNetModel on the host cores;
  * tests/test_final_latent_gpu.py : runs the reference fp32 and under bf16 autocast on the same GPU to measure the
    reference's OWN reduced-precision gap (the denominator of the final-latent tolerance, SURVEY 8d "Parity gate");
  * scripts/ref_gpu_compare.py : the reference's eager PyTorch-CUDA path as the honest comparator.

`mount()` makes `import ldm...`, `grounding_input...`, `inpaint_mask_func` resolve INSIDE the archive, in a way that
cannot be confused with this repo's drop-in modules of the same names: it must run in a process that has not imported
the repo's `ldm` (tests use a subprocess).
"""
from __future__ import annotations

import hashlib
import os
import sys
import zipfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
OUT_DIR = os.path.join(HERE, "_ref")
ZIP = os.path.join(OUT_DIR, "gligen_reference.zip")
# what the hot path (+ the VAE decoder, the next row) imports; everything else of the reference is out of scope
INCLUDE_DIRS = ["ldm", "grounding_input"]
INCLUDE_FILES = ["inpaint_mask_func.py", "convert_ckpt.py"]
DATA_FILES = ["SD_input_conv_weight_bias.pth"]          # read CWD-relative by restore_first_conv_from_SD (openaimodel.py:404)


def build() -> str:
    if not os.path.isdir(REF):
        if os.path.exists(ZIP):
            return ZIP
        raise RuntimeError(f"{REF} is absent and {ZIP} was not prebuilt")
    os.makedirs(OUT_DIR, exist_ok=True)
    names = []
    for d in INCLUDE_DIRS:
        for root, _, files in os.walk(os.path.join(REF, d)):
            for f in sorted(files):
                if f.endswith(".py"):
                    names.append(os.path.relpath(os.path.join(root, f), REF))
    names += INCLUDE_FILES
    names.sort()
    h = hashlib.sha256()
    with zipfile.ZipFile(ZIP + ".tmp", "w", zipfile.ZIP_DEFLATED) as z:
        for n in names:
            with open(os.path.join(REF, n), "rb") as f:
                data = f.read()
            h.update(n.encode()); h.update(data)
            zi = zipfile.ZipInfo(n, date_time=(2020, 1, 1, 0, 0, 0))      # reproducible archive
            zi.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(zi, data)
    os.replace(ZIP + ".tmp", ZIP)
    for n in DATA_FILES:
        with open(os.path.join(REF, n), "rb") as f, open(os.path.join(OUT_DIR, n), "wb") as g:
            g.write(f.read())
    with open(os.path.join(OUT_DIR, "MANIFEST.txt"), "w") as f:
        f.write(f"source {REF}\nfiles {len(names)}\nsha256 {h.hexdigest()}\n")
    return ZIP


def available() -> bool:
    return os.path.exists(ZIP)


def mount() -> str:
    """Route `ldm`, `grounding_input`, `inpaint_mask_func` imports of THIS process to the archived reference."""
    import importlib.machinery
    import types
    if not available():
        raise RuntimeError(f"{ZIP} is missing: run `python oracle/build_ref.py` where /root/reference exists")
    for name in ("ldm", "grounding_input"):
        if name in sys.modules and ZIP not in str(getattr(sys.modules[name], "__path__", "")):
            raise RuntimeError(f"`{name}` is already imported from {getattr(sys.modules[name], '__path__', '?')}: "
                               "mount the reference in a fresh process")
    if ZIP not in sys.path:
        sys.path.insert(0, ZIP)
    # `ldm` is a namespace package in the reference (no ldm/__init__.py) while this repo's drop-in `ldm` is a regular
    # package that would win the import whatever the sys.path order: pin the package to the archive explicitly.
    path = ZIP + "/ldm"
    spec = importlib.machinery.ModuleSpec("ldm", None, is_package=True)
    spec.submodule_search_locations = [path]
    mod = types.ModuleType("ldm")
    mod.__path__ = [path]
    mod.__spec__ = spec
    sys.modules["ldm"] = mod
    for sub in ("ldm.models", "ldm.modules"):                   # namespace levels of the reference tree
        p = ZIP + "/" + sub.replace(".", "/")
        s = importlib.machinery.ModuleSpec(sub, None, is_package=True)
        s.submodule_search_locations = [p]
        m = types.ModuleType(sub)
        m.__path__ = [p]
        m.__spec__ = s
        sys.modules[sub] = m
        setattr(sys.modules[sub.rsplit(".", 1)[0]], sub.rsplit(".", 1)[1], m)
    return OUT_DIR


if __name__ == "__main__":
    print(build())
