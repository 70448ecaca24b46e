"""Stages the original project's video drivers, illustrip.py and illustra.py, into oracle/_ref/ (git-ignored).

TEST INFRASTRUCTURE. tests/test_real_script_illustrip.py and tests/test_illustrip_host.py run the UNMODIFIED scripts through the
launcher, next to the `aphantasia/` package that stage_ref.stage() places there. The scripts belong to the original project and
are never committed here; build() calls stage() after stage_ref.stage(), so that copies sit beside the built library wherever the
reference tree (ref_import.REF_ROOT) is readable. Where it is not, earlier staged copies are kept as they are, and without them
those tests skip. Files are written with default permissions so that a later stage() can overwrite them.
"""
import os
import shutil

from oracle.ref_import import REF_ROOT
from oracle.stage_ref import STAGE

SCRIPTS = ('illustrip.py', 'illustra.py')


def stage():
    """Copies REF_ROOT/illustrip.py and REF_ROOT/illustra.py into oracle/_ref/. Returns the names staged now or earlier."""
    staged = []
    for name in SCRIPTS:
        src, dst = os.path.join(REF_ROOT, name), os.path.join(STAGE, name)
        if os.path.isfile(src) and os.access(src, os.R_OK):
            os.makedirs(STAGE, exist_ok=True)
            shutil.copyfile(src, dst)
        if os.path.isfile(dst):
            staged.append(name)
    return staged
