"""Compile the reference's OWN ``c_gae.pyx`` from a PufferLib source checkout.  TEST INFRASTRUCTURE.

The checkout is the directory named by the environment variable PUFFERLIB_REFERENCE (nothing is built without it).
Recipe (no reference build system involved): ``cython`` translates its c_gae.pyx to C in a temp dir, ``gcc``
compiles that one file into ``oracle/_ref/c_gae*.so`` (git-ignored).  Nothing is copied into the repo history.
``load()`` imports the built module if present; tests/golden/generate.py stores its outputs as golden data, so the
tests compare against the reference without it.
"""
import glob
import importlib.util
import os
import subprocess
import sys
import sysconfig
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, '_ref')


def reference_dir():
    """The PufferLib source checkout named by PUFFERLIB_REFERENCE, or None."""
    ref = os.environ.get('PUFFERLIB_REFERENCE')
    return ref if ref and os.path.exists(os.path.join(ref, 'c_gae.pyx')) else None


def build(force=False):
    existing = glob.glob(os.path.join(OUT, 'c_gae*.so'))
    if existing and not force:
        return existing[0]
    ref = reference_dir()
    if ref is None:
        return None
    src = os.path.join(ref, 'c_gae.pyx')
    import numpy as np
    os.makedirs(OUT, exist_ok=True)
    ext = sysconfig.get_config_var('EXT_SUFFIX')
    so = os.path.join(OUT, 'c_gae' + ext)
    with tempfile.TemporaryDirectory() as tmp:
        c_file = os.path.join(tmp, 'c_gae.c')
        subprocess.check_call([sys.executable, '-m', 'cython', '-3', src, '-o', c_file])
        subprocess.check_call(['gcc', '-O2', '-fPIC', '-shared', '-fwrapv', '-fno-strict-aliasing',
                               '-I', sysconfig.get_paths()['include'], '-I', np.get_include(),
                               '-DNPY_NO_DEPRECATED_API=NPY_1_7_API_VERSION', c_file, '-o', so])
    return so


def load():
    """Return the reference's compiled ``c_gae`` module, or None if it was never built."""
    found = glob.glob(os.path.join(OUT, 'c_gae*.so'))
    if not found:
        return None
    spec = importlib.util.spec_from_file_location('c_gae', found[0])
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == '__main__':
    print(build(force=True))
