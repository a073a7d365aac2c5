"""Every libwmd symbol is classified for the launch-checking harness (tests/launch_check.py): a launch whose entry point
has a checker, a pack, or a size / query function.  A new entry point cannot ship without one."""
import inspect
import os
import re

from wavelet_monodepth_b200 import (_lib, kitti_eval, kitti_gt, kitti_hints, kitti_inputs, kitti_loss, nyu_eval, nyu_inputs,
                                    nyu_loss, ops)

import launch_check as lc

TABLES = _lib.TABLES                    # every table _lib.load() binds
ALL_SIGNATURES = {k: v for table in TABLES for k, v in table.items()}


def test_every_symbol_is_classified():
    """SYMBOLS covers every table _lib.load() binds (wmd.h, wmd_eval.h, wmd_loss.h, wmd_loss_kitti.h, wmd_hints.h,
    wmd_inputs.h, wmd_inputs_nyu.h and wmd_gt.h, which test_abi / the oracle tests hold to the headers), and nothing
    else."""
    assert len(ALL_SIGNATURES) == sum(len(table) for table in TABLES)
    for table in (_lib.KITTI_LOSS_SIGNATURES, _lib.HINTS_SIGNATURES, _lib.INPUTS_SIGNATURES, _lib.NYU_INPUTS_SIGNATURES,
                  _lib.GT_SIGNATURES):
        assert table and any(t is table for t in TABLES)
    unclassified = sorted(set(ALL_SIGNATURES) - set(lc.SYMBOLS))
    assert not unclassified, "libwmd symbols without a launch checker / pack / query classification: %s" % unclassified
    assert not sorted(set(lc.SYMBOLS) - set(ALL_SIGNATURES))


def test_launches_and_packs_name_their_wrapped_entry_points():
    for sym, kind in lc.SYMBOLS.items():
        if kind == "query":
            continue
        role, entry = kind
        assert role in ("launch", "pack"), (sym, kind)
        assert entry in (lc.ENTRIES if role == "launch" else lc.PACKS), (sym, entry)
        assert hasattr(lc.Harness, lc.hook("_check_", entry) if role == "launch" else "_pack_" + entry), (sym, entry)
    assert len(set(lc.ENTRIES)) == len(lc.ENTRIES)
    assert len({lc.hook("_check_", e) for e in lc.ENTRIES}) == len(lc.ENTRIES)
    for owner, attr in lc.ENTRY_POINTS:
        assert callable(getattr(owner, attr)), (owner, attr)


def _functions(module):
    """(entry name, function) of the module's own functions and of the methods of the classes it defines"""
    for name, fn in inspect.getmembers(module, inspect.isfunction):
        if fn.__module__ == module.__name__:
            yield lc.entry_name(module, name), fn
    for _, cls in inspect.getmembers(module, inspect.isclass):
        if cls.__module__ != module.__name__:
            continue
        for name, fn in vars(cls).items():
            if inspect.isfunction(fn):
                yield lc.entry_name(cls, name), fn


def test_every_ops_function_that_calls_libwmd_is_wrapped():
    """A function or method of ops, nyu_loss, nyu_eval, kitti_eval, kitti_loss, kitti_hints, kitti_inputs, nyu_inputs or
    kitti_gt that reaches a launch or pack symbol directly is a checked entry point or a pack."""
    wrapped = set(lc.ENTRIES) | set(lc.PACKS)
    found = set()
    for module in (ops, nyu_loss, nyu_eval, kitti_eval, kitti_loss, kitti_hints, kitti_inputs, nyu_inputs, kitti_gt):
        for name, fn in _functions(module):
            src = inspect.getsource(fn)
            used = [s for s, k in lc.SYMBOLS.items() if k != "query" and ".%s(" % s in src]
            if used:
                assert name in wrapped, (module.__name__, name, used)
                found.add(name)
    # every wrapped entry point of the evaluation, loss and pipeline modules calls libwmd itself
    assert {lc.entry_name(o, a) for o, a in lc.EVAL_LOSS + lc.PIPELINES} <= found
    for entry in set(lc.CHECKED) | set(lc.PACKS):
        assert callable(getattr(ops, entry)), entry


def _cases():
    """the workloads of the two workload modules and the direct cases of test_gpu_launch_footprint"""
    import test_gpu_production_launches as tp
    import test_gpu_workload_launches as tw
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_gpu_launch_footprint.py")) as f:
        direct = set(re.findall(r'"(direct:\w+)"', f.read()))
    return set(tp.WORKLOADS) | set(tw.WORKLOADS) | direct


def test_every_launch_symbol_has_a_case_that_reaches_it():
    """REACH names, for every launch symbol, the workload or direct case that calls it (each GPU case asserts that it
    does), and only cases that exist"""
    launches = {s for s, k in lc.SYMBOLS.items() if k != "query" and k[0] == "launch"}
    assert set(lc.REACH) == launches, sorted(set(lc.REACH) ^ launches)
    cases = _cases()
    unknown = {s: c for s, c in lc.REACH.items() if c not in cases}
    assert not unknown, unknown


def test_writes_names_parameters_of_its_entry_points():
    """every WRITES entry is a wrapped entry point and every name in it one of that entry's parameters"""
    params = {lc.entry_name(o, a): inspect.signature(getattr(o, a)).parameters for o, a in lc.ENTRY_POINTS}
    for entry, names in lc.WRITES.items():
        assert entry in params, entry
        assert names and set(names) <= set(params[entry]), (entry, names, list(params[entry]))
