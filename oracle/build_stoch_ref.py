"""Build the UNMODIFIED reference Stochastic MuZero ctree into oracle/_ref/stochastic_mz_tree*.so with the recipe of
oracle/build_ref.py, linked with two shims.

TEST INFRASTRUCTURE ONLY, like oracle/build_ref.py.  It compiles ``stochastic_mz_tree -> ctree_stochastic_muzero``
(stochastic_mz_tree.pyx + .pxd, lib/cnode.cpp, cnode.h, common_lib) with that recipe's flags, paths and output directory;
oracle/build_ref.py itself is unchanged.  The module is deliberately NOT an entry of build_ref.MODULES: build_ref.build links
one shim only, so a build_ref.build_all(force=True) would overwrite the pinned module with one whose chance draws are not
reproducible.  The module is linked with oracle/rand_shim.c (PUCT
ties draw rand() % len(ties) after a wall-clock reseed, cnode.cpp:659, 726: pinned to the first maximum) and
oracle/random_device_shim.cc (each chance draw seeds std::mt19937 from std::random_device, cnode.cpp:622-623: pinned to the
value given to ``set_random_device``), so the unmodified sources are reproducible.
"""
import ctypes
import importlib.machinery
import importlib.util
import os
import subprocess
import sys
import sysconfig
import tempfile

from oracle import build_ref

NAME = "stochastic_mz_tree"
SUBDIR = "ctree_stochastic_muzero"
_mod = None


def build(force: bool = False) -> str:
    """Returns the path of the built module, or '' if the reference tree is absent."""
    target = build_ref.ref_module_path(NAME)
    if os.path.exists(target) and not force:
        return target
    src_dir = os.path.join(build_ref.CTREE, SUBDIR)
    if not os.path.isdir(src_dir):
        return ""
    import numpy
    os.makedirs(os.path.dirname(target), exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        gen_cpp = os.path.join(tmp, NAME + ".cpp")
        subprocess.check_call([sys.executable, "-m", "cython", "--cplus", "-3", "-I", src_dir,
                               os.path.join(src_dir, NAME + ".pyx"), "-o", gen_cpp])
        shims = [os.path.join(tmp, "rand_shim.o"), os.path.join(tmp, "random_device_shim.o")]
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-c", os.path.join(build_ref.HERE, "rand_shim.c"), "-o", shims[0]])
        subprocess.check_call(["g++", "-std=c++11", "-O2", "-fPIC", "-c", os.path.join(build_ref.HERE, "random_device_shim.cc"),
                               "-o", shims[1]])
        subprocess.check_call(["g++", "-std=c++11", "-O2", "-DNDEBUG", "-fPIC", "-shared", "-w",
                               "-I", sysconfig.get_paths()["include"], "-I", numpy.get_include(), "-I", src_dir,
                               "-I", os.path.join(src_dir, "lib"), "-I", build_ref.CTREE, gen_cpp] + shims + ["-o", target])
    return target


def load():
    """The compiled module, or None when it was not built (no reference sources)."""
    global _mod
    if _mod is None:
        path = build_ref.ref_module_path(NAME)
        if not os.path.exists(path):
            return None
        loader = importlib.machinery.ExtensionFileLoader(NAME, path)
        spec = importlib.util.spec_from_file_location(NAME, path, loader=loader)
        mod = importlib.util.module_from_spec(spec)
        loader.exec_module(mod)
        _mod = mod
    return _mod


def set_random_device(value: int):
    """What every std::random_device call of the loaded module returns from now on."""
    ctypes.CDLL(build_ref.ref_module_path(NAME)).lz_oracle_set_random_device(ctypes.c_uint(int(value) & 0xffffffff))


if __name__ == "__main__":
    print(build(force="--force" in sys.argv) or "reference tree not present; nothing built")
