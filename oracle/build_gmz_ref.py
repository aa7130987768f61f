"""Build the UNMODIFIED reference Gumbel MuZero ctree into oracle/_ref/gmz_tree*.so with the recipe of oracle/build_ref.py.

TEST INFRASTRUCTURE ONLY, like oracle/build_ref.py.  This file only registers one more entry of that recipe's MODULES table,
``gmz_tree -> ctree_gumbel_muzero`` (gmz_tree.pyx + .pxd, lib/cnode.cpp, cnode.h, common_lib), and calls its build();
oracle/build_ref.py itself is unchanged.  No rand() shim: the Gumbel search never calls rand() (cselect_child, the only
user, is not reached from cbatch_traverse) and its Gumbel vector comes from std::mt19937(0), so the module is
deterministic as built.
"""
import importlib.machinery
import importlib.util
import os
import sys

from oracle import build_ref

NAME = "gmz_tree"
build_ref.MODULES.setdefault(NAME, ("ctree_gumbel_muzero", False))


def build(force: bool = False) -> str:
    """Returns the path of the built module, or '' if the reference tree is absent."""
    return build_ref.build(force, NAME)


def load():
    """The compiled module, or None when it was not built (no reference sources)."""
    path = build_ref.ref_module_path(NAME)
    if not os.path.exists(path):
        return None
    loader = importlib.machinery.ExtensionFileLoader(NAME, path)
    spec = importlib.util.spec_from_file_location(NAME, path, loader=loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print(build(force="--force" in sys.argv) or "reference tree not present; nothing built")
