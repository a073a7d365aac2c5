"""Every libwmd symbol is classified for the launch-checking harness (tests/launch_check.py): a launch whose ops entry
point has a checker, a pack, or a size / query function.  A new entry point cannot ship without one."""
import inspect

from wavelet_monodepth_b200 import _lib, ops

import launch_check as lc


def test_every_symbol_is_classified():
    unclassified = sorted(set(_lib.SIGNATURES) - set(lc.SYMBOLS))
    assert not unclassified, "libwmd symbols without a launch checker / pack / query classification: %s" % unclassified
    assert not sorted(set(lc.SYMBOLS) - set(_lib.SIGNATURES))


def test_launches_and_packs_name_their_wrapped_entry_points():
    for sym, kind in lc.SYMBOLS.items():
        if kind == "query":
            continue
        role, entry = kind
        assert role in ("launch", "pack"), (sym, kind)
        assert entry in (lc.CHECKED if role == "launch" else lc.PACKS), (sym, entry)
        assert hasattr(lc.Harness, ("_check_" if role == "launch" else "_pack_") + entry), (sym, entry)


def test_every_ops_function_that_calls_libwmd_is_wrapped():
    """An ops function that reaches a launch or pack symbol directly is a checked entry point or a pack."""
    wrapped = set(lc.CHECKED) | set(lc.PACKS)
    for name, fn in inspect.getmembers(ops, inspect.isfunction):
        if fn.__module__ != ops.__name__:
            continue
        src = inspect.getsource(fn)
        used = [s for s, k in lc.SYMBOLS.items() if k != "query" and "lib.%s(" % s in src]
        if used:
            assert name in wrapped, (name, used)
    for entry in wrapped:
        assert callable(getattr(ops, entry)), entry
