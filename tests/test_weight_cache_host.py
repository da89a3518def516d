"""CPU: the cache of operands derived from parameters (``ops._derived_one`` / ``ops._derived``), exercised with CPU
parameters and a counting build function in place of the packing kernels."""
import gc
import importlib

import pytest
import torch
import torch.nn as nn

from e2fgvi_b200 import ops
from e2fgvi_b200.model.modules.feat_prop import SecondOrderDeformableAlignment


class CountingBuild:
    """Build function that records how often it ran and returns a copy of its parameters' values."""

    def __init__(self):
        self.calls = 0

    def __call__(self, *params):
        self.calls += 1
        return [p.detach().clone() for p in params]


def _param(seed, n=6):
    return nn.Parameter(torch.randn(n, generator=torch.Generator().manual_seed(seed)))


def test_hit_does_not_rebuild():
    p, q = _param(0), _param(1)
    build = CountingBuild()
    first = ops._derived_one(p, ("t", 1), build)
    assert ops._derived_one(p, ("t", 1), build) is first
    assert build.calls == 1
    ops._derived_one(p, ("t", 2), build)                               # another tag is another operand
    assert build.calls == 2
    pair = ops._derived([p, q], ("t", 1), lambda: build(p, q))
    assert ops._derived([p, q], ("t", 1), lambda: build(p, q)) is pair
    assert build.calls == 3


def test_rebuilt_after_in_place_update():
    p, q = _param(2), _param(3)
    build = CountingBuild()
    ops._derived_one(p, ("t",), build)
    ops._derived([p, q], ("t",), lambda: build(p, q))
    with torch.no_grad():
        p.mul_(2.0)                                                       # bumps p._version
    assert torch.equal(ops._derived_one(p, ("t",), build)[0], p.detach())
    assert build.calls == 3
    with torch.no_grad():
        q.add_(1.0)                                                       # any parameter of a multi-parameter entry
    got = ops._derived([p, q], ("t",), lambda: build(p, q))
    assert build.calls == 4 and torch.equal(got[0], p.detach()) and torch.equal(got[1], q.detach())


def test_rebuilt_after_data_assignment():
    p = _param(4)
    build = CountingBuild()
    ops._derived_one(p, ("t",), build)
    version = p._version
    p.data = torch.full((6,), 7.0)                                        # new storage, same version
    assert p._version == version
    assert torch.equal(ops._derived_one(p, ("t",), build)[0], torch.full((6,), 7.0))
    assert build.calls == 2


def test_rebuilt_when_a_new_parameter_reuses_a_dead_ones_id():
    storage = torch.arange(6.0)
    p = nn.Parameter(storage)        # aliases `storage`: its successor has the same version and data_ptr
    build = CountingBuild()
    ops._derived_one(p, ("t",), build)
    dead_id = id(p)
    del p
    gc.collect()
    kept = []
    for _ in range(1000):
        p2 = nn.Parameter(storage)
        if id(p2) == dead_id:
            break
        kept.append(p2)
    else:
        pytest.skip("the allocator never reused the dead parameter's id")
    ops._derived_one(p2, ("t",), build)
    assert build.calls == 2


def test_entry_dropped_when_the_parameter_is_collected():
    p, q = _param(5), _param(6)
    build = CountingBuild()
    ops._derived_one(p, ("t",), build)
    ops._derived([q, p], ("t",), lambda: build(q, p))
    one, pair = (id(p), ("t",)), ((id(q), id(p)), ("t",))
    assert one in ops._DERIVED and pair in ops._DERIVED
    del p
    gc.collect()
    assert one not in ops._DERIVED and pair in ops._DERIVED       # a list's entry lives with its first parameter
    del q
    gc.collect()
    assert pair not in ops._DERIVED


def test_invalidate_weight_caches_clears_everything():
    p, q = _param(7), _param(8)
    build = CountingBuild()
    ops._derived_one(p, ("t",), build)
    ops._derived([p, q], ("t",), lambda: build(p, q))
    ops.invalidate_weight_caches()
    assert not ops._DERIVED
    ops._derived_one(p, ("t",), build)
    ops._derived([p, q], ("t",), lambda: build(p, q))
    assert build.calls == 4


@pytest.fixture
def counting_dcn_pack(monkeypatch):
    calls = []

    def pack(weight, deform_groups):                                      # CPU stand-in for the packing kernel
        calls.append(deform_groups)
        return weight.detach().clone()

    monkeypatch.setattr(ops, "pack_dcn_weight", pack)
    return calls


def test_dcn_packed_weight_follows_load_state_dict(counting_dcn_pack):
    m = SecondOrderDeformableAlignment(32, 16, 3, padding=1, deform_groups=2)
    first = m.packed_weight()
    assert m.packed_weight() is first and counting_dcn_pack == [2]
    sd = {k: v + 1.0 for k, v in m.state_dict().items()}
    m.load_state_dict(sd)
    assert torch.equal(m.packed_weight(), sd["weight"]) and len(counting_dcn_pack) == 2


def test_generator_invalidates_the_dcn_operand(counting_dcn_pack):
    """``.data`` updates bump no version: ``init_weights`` and ``load_state_dict`` of the generator drop the packed
    DCN weight with every other derived operand."""
    model = importlib.import_module("model.e2fgvi").InpaintGenerator()
    align = model.feat_prop_module.deform_align["backward_"]
    align.packed_weight()
    align.weight.data.copy_(torch.ones_like(align.weight))
    model.init_weights()
    assert torch.equal(align.packed_weight(), torch.ones_like(align.weight)) and len(counting_dcn_pack) == 2
    sd = model.state_dict()
    sd["feat_prop_module.deform_align.backward_.weight"] = torch.zeros_like(align.weight)
    model.load_state_dict(sd)
    assert float(align.packed_weight().abs().max()) == 0.0 and len(counting_dcn_pack) == 3
