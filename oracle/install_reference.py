"""Recipe that installs the UNMODIFIED original project (ckczzj/PDAE) into oracle/_ref (git-ignored), for
`bench.py --impl reference` and the drop-in test.  Called by `__graft_entry__.build()`.

The sources are looked up in $PDAE_REFERENCE_DIR, else in a checkout named `reference` beside this repository.  Without
them nothing is installed and the users of oracle/_ref fall back (bench) or skip (drop-in test).  The original project is
a flat Python repo without setup.py / pyproject.toml, so the install is what its own scripts do -- PYTHONPATH=<repo root>
-- i.e. a copy of its package directories.  Nothing under oracle/_ref is product source, and none of it is committed."""
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
PACKAGES = ("model", "diffusion", "metric", "sampler", "trainer", "dataset", "utils", "config")


def source_dir() -> str:
    return os.environ.get("PDAE_REFERENCE_DIR") or os.path.join(os.path.dirname(ROOT), "reference")


def install() -> str:
    src_root = source_dir()
    if not os.path.isfile(os.path.join(src_root, "model", "shift_unet.py")) or not os.access(src_root, os.R_OK | os.X_OK):
        return "prebuilt" if os.path.isdir(REF_DIR) else "absent"
    os.makedirs(REF_DIR, exist_ok=True)
    for pkg in PACKAGES:
        src, dst = os.path.join(src_root, pkg), os.path.join(REF_DIR, pkg)
        if os.path.isdir(src):
            shutil.rmtree(dst, ignore_errors=True)
            shutil.copytree(src, dst, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    with open(os.path.join(REF_DIR, "INSTALL_NOTE.txt"), "w") as f:
        f.write(f"ckczzj/PDAE package directories {PACKAGES}, copied unmodified\n")
    return "installed"
