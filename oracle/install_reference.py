#!/usr/bin/env python
"""Install the UNMODIFIED reference MUSt3R checkout under oracle/_ref (git-ignored).

    [MUST3R_REFERENCE=<reference checkout>] python oracle/install_reference.py

The checkout is $MUST3R_REFERENCE if set, else the first of SEARCH that exists: a `reference` directory beside this
repository, then /root/reference, where the reference checkout of the build environment lives.  Without one there is
nothing to install and the callers below skip or fall back.

Used by `bench.py --impl reference` (the CPU arm drives the reference's own engine), bench.py's parity record and the
GPU seam test of the reference's import-time RoPE selection; everything else runs without it.  Recipe: `pip install
--no-index --no-build-isolation --no-deps --target oracle/_ref <copy of the checkout>` (a temporary copy because the
build writes egg-info into the source tree; --no-deps because its requirements - gradio, open3d, viser, roma, git+https
dependencies - cannot be resolved offline).  setup.py only packages `must3r`; its `dust3r` / `croco` dependencies are
git submodules of the checkout, which must3r finds by relative path (must3r/tools/path_to_dust3r.py), so their python
packages are placed next to it with the same layout.  Nothing is edited; INSTALL.json records a sha256 per file so
tests can prove the copy is byte-identical to what this script read.
"""
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEARCH = [os.path.join(os.path.dirname(ROOT), "reference"), "/root/reference"]


def _is_checkout(d):
    try:
        return os.path.isfile(os.path.join(d, "setup.py")) and os.path.isdir(os.path.join(d, "must3r"))
    except OSError:
        return False


def source():
    """The reference checkout to install from, or None."""
    env = os.environ.get("MUST3R_REFERENCE")
    if env:
        return env if _is_checkout(env) else None
    return next((d for d in SEARCH if _is_checkout(d)), None)


SRC = source()
DST = os.path.join(ROOT, "oracle", "_ref")
SUBMODULE_DIRS = ["dust3r/dust3r", "dust3r/croco/models", "dust3r/croco/utils"]


def main():
    if SRC is None:
        print("no reference checkout found ($MUST3R_REFERENCE or " + ", ".join(SEARCH) + "): nothing to install")
        return 0
    shutil.rmtree(DST, ignore_errors=True)
    os.makedirs(DST)
    tmp = tempfile.mkdtemp(prefix="m3r_ref_src_")
    shutil.copytree(os.path.join(SRC, "must3r"), os.path.join(tmp, "must3r"))
    shutil.copy(os.path.join(SRC, "setup.py"), tmp)
    cmd = [sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps", "--target", DST, tmp]
    r = subprocess.run(cmd, capture_output=True, text=True)
    shutil.rmtree(tmp, ignore_errors=True)
    pip_ok = r.returncode == 0 and os.path.isdir(os.path.join(DST, "must3r"))
    note = "pip install --target ok" if pip_ok else f"pip failed (rc {r.returncode}): {(r.stderr or r.stdout).strip().splitlines()[-1:]}; plain copy used"
    if not pip_ok:
        shutil.rmtree(os.path.join(DST, "must3r"), ignore_errors=True)
        shutil.copytree(os.path.join(SRC, "must3r"), os.path.join(DST, "must3r"))
    for d in SUBMODULE_DIRS:
        shutil.copytree(os.path.join(SRC, d), os.path.join(DST, d), ignore=shutil.ignore_patterns("*.so", "build", "__pycache__"))
    files = {}
    for base, _, names in os.walk(DST):
        for n in names:
            if n.endswith((".py", ".cu", ".cpp")) and "dist-info" not in base:
                p = os.path.join(base, n)
                rel = os.path.relpath(p, DST)
                src = os.path.join(SRC, rel)
                h = hashlib.sha256(open(p, "rb").read()).hexdigest()
                same = os.path.exists(src) and hashlib.sha256(open(src, "rb").read()).hexdigest() == h
                files[rel] = {"sha256": h, "identical_to_reference": same}
    bad = [k for k, v in files.items() if not v["identical_to_reference"]]
    json.dump({"source": SRC, "method": note, "n_files": len(files), "modified": bad, "files": files},
              open(os.path.join(DST, "INSTALL.json"), "w"), indent=1)
    print(f"oracle/_ref: {len(files)} source files, {note}; files differing from {SRC}: {bad or 'none'}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
