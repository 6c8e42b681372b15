"""Vendors the UNMODIFIED reference (Samsung/veles.znicz) into ``oracle/_ref/veles/znicz``
(git-ignored; ``__graft_entry__.build()`` runs this where the reference source tree exists, and
the reference arm of ``bench.py`` and ``tests/test_reference_arm.py`` use what it installed).

``pip install --target oracle/_ref <reference tree>`` cannot work (the tree has neither
setup.py nor pyproject.toml: it is a plugin directory of the Veles platform), so the files
are copied byte for byte (bulky test data, docs and the C++ libZnicz are skipped) and a
sha256 manifest is written next to them: ``verify()`` proves nothing was edited.
The absent Veles core itself (package ``veles``: units, workflow, memory, loaders, NVRTC
build, ...), ``cuda4py`` and ``zope.interface`` are supplied by ``baseline/veles_core``.
"""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, "_ref", "veles", "znicz")
# where the reference source tree is read from (ZNICZ_REFERENCE overrides)
SRC = os.environ.get("ZNICZ_REFERENCE", "/root/reference")
SKIP_DIRS = {"tests", "docs", "libZnicz", ".git", "__pycache__"}


def _sha(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 20), b""):
            h.update(blk)
    return h.hexdigest()


def install(src=SRC, force=False):
    if os.path.isfile(os.path.join(DST, "MANIFEST.sha256.json")) and not force:
        return DST
    if not os.path.isdir(src):
        raise RuntimeError("reference tree %s not found" % src)
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    manifest = {}
    for dirpath, dirnames, filenames in os.walk(src):
        rel = os.path.relpath(dirpath, src)
        parts = [] if rel == "." else rel.split(os.sep)
        if parts and parts[0] in SKIP_DIRS:
            dirnames[:] = []
            continue
        dirnames[:] = [d for d in dirnames if d not in SKIP_DIRS or parts]
        out = os.path.join(DST, *parts)
        os.makedirs(out, exist_ok=True)
        for fn in filenames:
            s = os.path.join(dirpath, fn)
            d = os.path.join(out, fn)
            shutil.copyfile(s, d)
            manifest[os.path.join(*parts, fn) if parts else fn] = _sha(d)
    with open(os.path.join(DST, "MANIFEST.sha256.json"), "w") as f:
        json.dump(manifest, f, indent=0, sort_keys=True)
    return DST


def verify(src=None):
    """Every vendored file still has the hash recorded at install time (and equals the
    file under ``src`` when the reference tree is mounted)."""
    with open(os.path.join(DST, "MANIFEST.sha256.json")) as f:
        manifest = json.load(f)
    bad = []
    for rel, h in manifest.items():
        p = os.path.join(DST, rel)
        if not os.path.isfile(p) or _sha(p) != h:
            bad.append(rel)
        elif src and os.path.isfile(os.path.join(src, rel)) and _sha(os.path.join(src, rel)) != h:
            bad.append(rel)
    return bad


if __name__ == "__main__":
    print(install(force="--force" in sys.argv))
    print("modified files:", verify(SRC))
