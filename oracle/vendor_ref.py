"""Recipe that vendors the UNMODIFIED reference for the CPU arm of bench.py: copies the four source directories of the
general_cf path (config/ data_utils/ models/ trainer/, ~0.8 MB, no datasets) from the reference checkout
($SSLREC_REFERENCE, by default /root/reference) into oracle/_ref/.
TEST / BASELINE INFRASTRUCTURE ONLY.

oracle/_ref/ is git-ignored (the reference's sources never enter this repository's history); it stays next to the
working tree, so a copy of the tree carries it to a machine without the reference checkout.  Users: ``bench.py --impl
reference`` (the CPU arm runs the reference's own code, ``kind: "reference"``; without oracle/_ref, the oracle port) and
tests/test_dropin_reference.py (the reference's build_data_handler / build_model / Trainer / Metric driving this
repository's models through the INTEGRATION.md shims; skipped without oracle/_ref).  ``__graft_entry__.build()`` runs
this whenever the reference checkout is present.  The product package never imports anything from here.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get('SSLREC_REFERENCE', '/root/reference')
DST = os.path.join(HERE, '_ref')
DIRS = ('config', 'data_utils', 'models', 'trainer')


def available() -> bool:
    return all(os.path.isdir(os.path.join(DST, d)) for d in DIRS)


def vendor(force: bool = False) -> str:
    if not os.path.isdir(REF):
        if available():
            return DST
        raise FileNotFoundError(f'{REF} not found and {DST} is empty: set SSLREC_REFERENCE to a reference checkout')
    if available() and not force:
        return DST
    for d in DIRS:
        dst = os.path.join(DST, d)
        if os.path.isdir(dst):
            shutil.rmtree(dst)
        shutil.copytree(os.path.join(REF, d), dst, ignore=shutil.ignore_patterns('__pycache__', '*.pyc'))
    # manifest: file list + digest, so a test can state which reference revision it ran
    h = hashlib.sha256()
    names = []
    for d in DIRS:
        for root, _, files in sorted(os.walk(os.path.join(DST, d))):
            for f in sorted(files):
                p = os.path.join(root, f)
                names.append(os.path.relpath(p, DST))
                h.update(open(p, 'rb').read())
    with open(os.path.join(DST, 'MANIFEST.txt'), 'w') as f:
        f.write(f'source: {REF}\nsha256(all files): {h.hexdigest()}\nfiles: {len(names)}\n' + '\n'.join(names) + '\n')
    return DST


if __name__ == '__main__':
    print(vendor(force='--force' in sys.argv))
