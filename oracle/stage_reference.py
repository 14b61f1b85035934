"""Stage the reference's own model modules into the git-ignored ``oracle/_ref/`` (run by ``__graft_entry__.build()``).

The reference (ruizhecao96/CMGAN) is a plain source tree without packaging, so the four files its model code consists of --
models/generator.py, models/conformer.py, models/discriminator.py, utils.py -- are copied unmodified from the checkout named by
``CMGAN_REFERENCE`` (default ``/root/reference``).  ``bench.py``'s reference arms import them from ``oracle/_ref/``; where neither a
checkout nor a staged copy exists they fall back to the oracle port and say so (``kind: "port"``).  Nothing under ``oracle/_ref/``
is tracked, and the ``cmgan_b200`` package never imports it.
"""
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref")
FILES = ["models/generator.py", "models/conformer.py", "models/discriminator.py", "utils.py"]


def stage() -> bool:
    """copy the reference modules into oracle/_ref; False (and nothing touched) when no reference checkout is present"""
    src = os.path.join(os.environ.get("CMGAN_REFERENCE", "/root/reference"), "src")
    if not all(os.path.isfile(os.path.join(src, f)) for f in FILES):
        return False
    for f in FILES:
        d = os.path.join(DST, f)
        os.makedirs(os.path.dirname(d), exist_ok=True)
        shutil.copyfile(os.path.join(src, f), d)
    return True


if __name__ == "__main__":
    print("staged into " + DST if stage() else "no reference checkout found: nothing staged")
