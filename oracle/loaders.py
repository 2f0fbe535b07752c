"""ctypes loaders of the two CPU oracles -- TEST INFRASTRUCTURE: only tests/, __graft_entry__.smoke() and bench.py's reference leg
may import this module; the product package (miniasm_b200/) never does.

* ``load_reference()``   -> oracle/_ref/libminiasm_ref.so, the UNMODIFIED reference compiled by oracle/Makefile
* ``load_oracle_port()`` -> oracle/libma_oracle.so, our sequential C restatement (oracle/ma_oracle.c)

Both export the reference's own C API, so the ctypes bindings of the product (miniasm_b200.capi.Lib) drive them too.
"""
import os
import re

from miniasm_b200.capi import Lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE_SO = os.path.join(ROOT, "oracle", "_ref", "libminiasm_ref.so")
# the reference's source tree: oracle/Makefile's REF (overridable from the environment, as for make)
REFERENCE_SRC = os.environ.get("REF") or re.search(r"^REF\s*\?=\s*(\S+)", open(os.path.join(ROOT, "oracle", "Makefile")).read(), re.M).group(1)
ORACLE_SO = os.path.join(ROOT, "oracle", "libma_oracle.so")


def load_reference():
    return Lib(REFERENCE_SO, product=False, strict=True)


def load_oracle_port():
    return Lib(ORACLE_SO, product=False, strict=False)
