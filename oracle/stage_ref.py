"""Stages the original project's clip_fft.py and its `aphantasia/` package into oracle/_ref/ (git-ignored).

TEST INFRASTRUCTURE. The end-to-end tests run the UNMODIFIED script through the launcher (tests/test_real_script.py,
tests/test_host.py::test_launcher_runs_the_real_clip_fft_imports). The script belongs to the original project and is never
committed here; build() calls stage() so that a copy sits beside the built library wherever the reference tree
(ref_import.REF_ROOT) is readable. Where it is not, an earlier staged copy is kept as it is, and without one those tests skip.
Files are written with default permissions so that a later stage() can overwrite them.
"""
import os
import shutil

from oracle.ref_import import REF_ROOT

STAGE = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_ref')


def stage():
    """Copies REF_ROOT/clip_fft.py and REF_ROOT/aphantasia/ into oracle/_ref/. Returns the staged tree, or None."""
    script = os.path.join(REF_ROOT, 'clip_fft.py')
    if not (os.path.isfile(script) and os.access(script, os.R_OK)):
        return STAGE if os.path.isfile(os.path.join(STAGE, 'clip_fft.py')) else None
    os.makedirs(STAGE, exist_ok=True)
    shutil.copyfile(script, os.path.join(STAGE, 'clip_fft.py'))
    pkg = os.path.join(REF_ROOT, 'aphantasia')
    for d, dirs, files in os.walk(pkg):
        dirs[:] = [x for x in dirs if x != '__pycache__']
        out = os.path.join(STAGE, 'aphantasia', os.path.relpath(d, pkg))
        os.makedirs(out, exist_ok=True)
        for f in files:
            shutil.copyfile(os.path.join(d, f), os.path.join(out, f))
    return STAGE
