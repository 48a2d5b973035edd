#!/usr/bin/env python
"""Recipe that installs the UNMODIFIED reference (reczoo/FuxiCTR) under oracle/_ref/, the checker that the
reference-boundary tests, the live-reference comparisons and bench.py's reference arms run against.
`__graft_entry__.build()` calls install(); by hand:

    python oracle/install_ref.py [--force]

The reference checkout is read from $FUXICTR_REFERENCE (default /root/reference).  When it is absent, an
oracle/_ref/ installed earlier is kept as it is (a copy of the tree made after the build carries it along),
and without either the tests that need the reference skip.

1. `pip install --no-index --no-build-isolation --no-deps --target oracle/_ref <copy of the checkout>` — the
   `fuxictr` package exactly as setup.py ships it.  (--no-deps: keras_preprocessing, h5py and polars are
   import-time-only on this path and stubbed by baseline/refenv.py, SURVEY.md 8c.  The copy in a temporary
   directory is needed because setup.py writes build/ and *.egg-info into its source tree.)
2. What setup.py does NOT package but the reference's own entry points read at run time, copied verbatim into
   oracle/_ref/extras/: the five in-scope `model_zoo` directories (run_expid.py + config/*.yaml + src/),
   `demo/` (example3 = BASELINE config C1) and the `data/tiny_*` fixtures those YAMLs point at.

oracle/_ref is git-ignored: nothing under it is product source or enters history.
"""
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("FUXICTR_REFERENCE", "/root/reference")
DST = os.path.join(HERE, "_ref")
STAMP = os.path.join(DST, "INSTALLED")
ZOO = ["DeepFM", "DCNv2", "DLRM", "DIN", "xDeepFM"]
DATA = ["tiny_npz", "tiny_parquet", "tiny_seq", "tiny_csv"]


def installed():
    return os.path.exists(STAMP)


def install(force=False):
    """Install the reference into oracle/_ref unless it is already there.  Returns True when oracle/_ref
    holds a complete install afterwards, False when there is neither an install nor a reference to make one."""
    if installed() and not force:
        return True
    if not os.path.isdir(os.path.join(REF, "fuxictr")):
        return False
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "reference")
        shutil.copytree(REF, src, ignore=shutil.ignore_patterns(".git", "docs"))
        os.chmod(src, os.stat(src).st_mode | 0o700)
        for root, dirs, files in os.walk(src):     # the checkout may be read-only; setup.py writes into the copy
            for name in dirs + files:
                path = os.path.join(root, name)
                if not os.path.islink(path):
                    os.chmod(path, os.stat(path).st_mode | 0o200)
        cmd = [sys.executable, "-m", "pip", "install", "--quiet", "--no-index", "--no-build-isolation", "--no-deps",
               "--no-cache-dir", "--disable-pip-version-check", "--target", DST, src]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            shutil.rmtree(DST, ignore_errors=True)
            sys.stderr.write("oracle/install_ref.py: installing the reference from %s failed; the tests that "
                             "compare with it will skip:\n%s\n" % (REF, r.stdout[-4000:]))
            return False
    extras = os.path.join(DST, "extras")
    for name in ZOO:
        shutil.copytree(os.path.join(REF, "model_zoo", name), os.path.join(extras, "model_zoo", name))
    shutil.copytree(os.path.join(REF, "demo"), os.path.join(extras, "demo"))
    for name in DATA:
        shutil.copytree(os.path.join(REF, "data", name), os.path.join(extras, "data", name))
    for root, dirs, _ in os.walk(DST):
        for d in list(dirs):
            if d == "__pycache__":
                shutil.rmtree(os.path.join(root, d))
                dirs.remove(d)
    with open(STAMP, "w") as fd:
        fd.write(REF + "\n")
    return True


if __name__ == "__main__":
    if not install(force="--force" in sys.argv):
        raise SystemExit("no reference checkout at %s (set FUXICTR_REFERENCE)" % REF)
    print("installed the reference under", DST)
