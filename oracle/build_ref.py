"""Byte-compiled copy of the UNMODIFIED reference for the drop-in test and the CPU baseline arm.

`build()` (``__graft_entry__.py``) calls :func:`build_reference`: the reference's own ``main.py``, ``objective.py`` and
``optimizers/*.py`` are compiled to sourceless ``.pyc`` files under ``oracle/_ref/`` (git-ignored; no reference source
enters this repository).  Python imports them from there like the originals; the reference's missing ``helpers`` /
``datasets`` / ``tree`` submodules come from ``oracle/ref_shims``.  Where no reference checkout exists (a machine that
only runs the tests), an ``oracle/_ref/`` made earlier is kept as it is.
"""
import os
import py_compile

HERE = os.path.dirname(os.path.abspath(__file__))
REF_OUT = os.path.join(HERE, "_ref")
# checkout of jramapuram/BYOL the golden vectors were made from (tests/golden/make_golden.py); override with BYOL_REFERENCE
REFERENCE = os.environ.get("BYOL_REFERENCE", "/root/reference")
MODULES = ["main.py", "objective.py", "optimizers/lars.py", "optimizers/scheduler.py"]


def available():
    """True when oracle/_ref holds the compiled reference step loop."""
    return os.path.exists(os.path.join(REF_OUT, "main.pyc"))


def build_reference(reference=REFERENCE):
    """Compile the reference modules into oracle/_ref; returns True if oracle/_ref is usable afterwards."""
    if not os.path.exists(os.path.join(reference, "main.py")):
        return available()
    for rel in MODULES:
        src = os.path.join(reference, rel)
        if not os.path.exists(src):
            continue
        dst = os.path.join(REF_OUT, rel[:-3] + ".pyc")
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if os.path.exists(dst) and os.path.getmtime(dst) >= os.path.getmtime(src):
            continue
        py_compile.compile(src, cfile=dst, dfile=rel, doraise=True,
                           invalidation_mode=py_compile.PycInvalidationMode.UNCHECKED_HASH)
    return available()
