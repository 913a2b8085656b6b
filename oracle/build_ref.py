"""
Recipe for oracle/_ref/ -- TEST INFRASTRUCTURE ONLY (git-ignored, never part of the product path).

The reference's implementation of the hot path is one pure-Python file, tangram/mapping_optimizer.py of a
checkout of the original Tangram project (imports numpy, logging, torch only: lines 9-12).  There is nothing to
compile; to let the UNMODIFIED reference run next to this package, this script copies that one file verbatim into
oracle/_ref/ next to a stamp with its sha256.  The checkout is looked for next to this repository (../reference); the
TANGRAM_REFERENCE environment variable names another one.  oracle/_ref/ is listed in .gitignore (the reference's source
never enters this repo's history); once made, the copy serves where no checkout exists.

Users (and only these): bench.py's reference arms (`--impl reference` on the host cores; the `reference_gpu`
comparator with device='cuda'); bench.py reports those legs as skipped, with the reason, when no copy exists.

    python oracle/build_ref.py        # no-op without a checkout (uses the existing copy)
"""
import hashlib
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("TANGRAM_REFERENCE") or os.path.join(os.path.dirname(os.path.dirname(HERE)), "reference")
REF_SRC = os.path.join(REF_ROOT, "tangram", "mapping_optimizer.py")
REF_DIR = os.path.join(HERE, "_ref")
REF_DST = os.path.join(REF_DIR, "mapping_optimizer.py")
STAMP = os.path.join(REF_DIR, "SOURCE.txt")


def build():
    """Copy the reference file if the reference tree is present.  Returns the path of the copy or None."""
    if os.path.exists(REF_SRC):
        os.makedirs(REF_DIR, exist_ok=True)
        shutil.copyfile(REF_SRC, REF_DST)
        with open(REF_DST, "rb") as f:
            digest = hashlib.sha256(f.read()).hexdigest()
        with open(STAMP, "w") as f:
            f.write(f"verbatim copy of {REF_SRC}\nsha256 {digest}\n")
    return REF_DST if os.path.exists(REF_DST) else None


def _path():
    return REF_DST if os.path.exists(REF_DST) else (REF_SRC if os.path.exists(REF_SRC) else None)


def source():
    """Which file load() runs: {"path", "sha256"}, or None when there is neither a copy nor a checkout."""
    path = _path()
    if path is None:
        return None
    with open(path, "rb") as f:
        return {"path": path, "sha256": hashlib.sha256(f.read()).hexdigest()}


def load():
    """The unmodified reference module (classes Mapper, MapperConstrained), loaded by path."""
    import importlib.util
    path = _path()
    if path is None:
        raise FileNotFoundError("oracle/_ref/mapping_optimizer.py is missing: run `python oracle/build_ref.py` with a "
                                "Tangram checkout next to this repository or named by TANGRAM_REFERENCE")
    spec = importlib.util.spec_from_file_location("tangram_reference_mapping_optimizer", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print(build() or "no reference tree and no existing copy")
