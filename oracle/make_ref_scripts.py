#!/usr/bin/env python
"""Recipe: stage the UNMODIFIED reference's top-level `test.py` under oracle/_ref/ next to what oracle/make_ref.py stages.

    python oracle/make_ref_scripts.py    # build container only: /root/reference/test.py -> oracle/_ref/test.py

TEST INFRASTRUCTURE ONLY.  tests/test_gpu_loader.py loads the script from its file path (the stdlib has a `test`
package) and runs its `evaluate(model, test_loader)` over an installed AudioDataLoader on the GPU; only the functions are
used, its `__main__` block never runs.  Byte for byte, from the same source make_ref uses; oracle/_ref/ stays out of
git.  `__graft_entry__.build()` calls stage() after make_ref.stage().
"""
import filecmp
import os
import shutil
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import make_ref  # noqa: E402

SCRIPTS = ["test.py"]


def stage(verbose=True):
    """Copy SCRIPTS of make_ref.SRC into oracle/_ref/ (idempotent).  Returns the number staged, 0 if SRC is absent."""
    if not os.path.isdir(os.path.join(make_ref.SRC, "models", "asr")):
        return 0
    n = 0
    for rel in SCRIPTS:
        s, d = os.path.join(make_ref.SRC, rel), os.path.join(make_ref.DST, rel)
        if os.path.exists(s):
            os.makedirs(os.path.dirname(d), exist_ok=True)
            if not (os.path.exists(d) and filecmp.cmp(s, d, shallow=False)):
                shutil.copyfile(s, d)
            n += 1
    if verbose:
        print(f"make_ref_scripts: {n} script(s) of the unmodified reference staged in {make_ref.DST}")
    return n


if __name__ == "__main__":
    sys.exit(0 if stage() >= 0 else 1)
