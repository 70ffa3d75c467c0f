"""The ctypes mirrors of the sparse-group descriptors (`ops.GroupGeom`, `LookupTable`,
`PushTable`, `OwnerTable`) are checked against the layout the native library reports
(`px_sparse_abi`) when it loads.  Loading needs no GPU."""
import ctypes

import pytest

from parallax_b200 import ops
from parallax_b200.ops.build import nvcc

pytestmark = pytest.mark.skipif(nvcc() is None, reason="needs nvcc to build the library")


def test_library_layout_matches_ctypes():
    ops.lib()
    abi = ops.sparse_abi()
    assert abi["group_max"] == 4
    for cls in (ops.GroupGeom, ops.LookupTable, ops.PushTable, ops.OwnerTable):
        ops.check_struct(cls, abi)


def _push_table(fields):
    return type("PushTable", (ctypes.Structure,), {"_fields_": fields})


# dropping the last field (`scale`) leaves the size unchanged: only the field list notices
@pytest.mark.parametrize("drop", [f for f, _ in ops.PushTable._fields_])
def test_check_rejects_missing_field(drop):
    broken = _push_table([(f, t) for f, t in ops.PushTable._fields_ if f != drop])
    with pytest.raises(RuntimeError, match=r"PushTable\.%s\b.*rebuild" % drop):
        ops.check_struct(broken, ops.sparse_abi())


def test_check_rejects_extra_trailing_field():
    broken = _push_table(ops.PushTable._fields_ + [("extra", ctypes.c_int)])
    with pytest.raises(RuntimeError, match=r"PushTable\.extra\b.*rebuild"):
        ops.check_struct(broken, ops.sparse_abi())
