"""resize and table_occupancy call ctmr_resize / ctmr_group_resize and ctmr_table_occupancy / ctmr_group_table_occupancy
with their scalar arguments, None mapping to 0 (keep the size).  No GPU: test_binding_forms' fake library."""
import ctypes as C

import pytest

from test_binding_forms import _ctx, _group


@pytest.mark.parametrize("form", [_ctx, _group], ids=["ctx", "group"])
@pytest.mark.parametrize("args,want", [
    ((), (0, 0, 0)),
    ((1 << 25,), (1 << 25, 0, 0)),
    ((None, 26), (0, 26, 0)),
    ((None, None, 22), (0, 0, 22)),
    ((1000, 20, 18), (1000, 20, 18)),
])
def test_resize(form, args, want):
    db, lib, handles, prefix = form()
    db.resize(*args)
    assert [(n, a[0].value) for n, a in lib.calls] == [(prefix + "resize", handles["self"])]
    assert lib.calls[0][1][1:] == want


def test_resize_keywords():
    db, lib, _, _ = _ctx()
    db.resize(meta_capacity_log2=21, table_capacity=1 << 30)
    assert lib.calls[0][1][1:] == (1 << 30, 0, 21)


@pytest.mark.parametrize("form", [_ctx, _group], ids=["ctx", "group"])
def test_table_occupancy(form):
    db, lib, handles, prefix = form()
    used, cap = db.table_occupancy()
    assert [(n, a[0].value) for n, a in lib.calls] == [(prefix + "table_occupancy", handles["self"])]
    assert used == (0, 0, 0) and cap == (0, 0, 0)   # the fake library writes nothing
    _, u, c = lib.calls[0][1]
    assert isinstance(u, C.Array) and len(u) == 3 and isinstance(c, C.Array) and len(c) == 3
