"""Recipe of the reference install ``oracle/_ref`` that ``bench.py --impl reference`` runs (git-ignored build product).

``__graft_entry__.build()`` runs it when the reference source tree is present (``D9D_REFERENCE_SRC``, by default
``/root/reference``); the result stays next to the build, so a machine that only receives the built tree can still run
the reference arm.  A wheel install is not possible offline (the reference's PEP-517 backend ``poetry-core`` is not
installable without an index), and the package is pure Python, so what a wheel install would have produced is a
verbatim copy of ``d9d/`` plus a ``dist-info``: this recipe makes exactly that (byte-for-byte copy, sha256 ``RECORD`` so
the copy can be audited against its source) and also copies ``example/`` (the benchmark drives the example's own
providers).
"""

from __future__ import annotations

import base64
import hashlib
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DEST = os.path.join(HERE, "_ref")


def install(src: str = os.environ.get("D9D_REFERENCE_SRC", "/root/reference"), dest: str = DEST) -> bool:
    if not os.path.isdir(os.path.join(src, "d9d")):
        return False
    os.makedirs(dest, exist_ok=True)
    for sub in ("d9d", "example"):
        target = os.path.join(dest, sub)
        if os.path.isdir(target):
            shutil.rmtree(target)
        shutil.copytree(os.path.join(src, sub), target, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    info = os.path.join(dest, "d9d-0.14.0.dist-info")
    os.makedirs(info, exist_ok=True)
    with open(os.path.join(info, "METADATA"), "w") as f:
        f.write("Metadata-Version: 2.1\nName: d9d\nVersion: 0.14.0\nSummary: verbatim copy of the reference's d9d package (poetry-core unavailable offline)\n")
    with open(os.path.join(info, "INSTALLER"), "w") as f:
        f.write("oracle/install_reference.py\n")
    records = []
    for root, _dirs, files in os.walk(os.path.join(dest, "d9d")):
        for name in sorted(files):
            path = os.path.join(root, name)
            with open(path, "rb") as fh:
                data = fh.read()
            digest = base64.urlsafe_b64encode(hashlib.sha256(data).digest()).rstrip(b"=").decode()
            records.append(f"{os.path.relpath(path, dest)},sha256={digest},{len(data)}")
    with open(os.path.join(info, "RECORD"), "w") as f:
        f.write("\n".join(sorted(records)) + "\n")
    return True


if __name__ == "__main__":
    ok = install(*sys.argv[1:2])
    print("installed" if ok else "reference source not found", DEST)
