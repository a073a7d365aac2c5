"""ops._launch, the one path from Python into libwmd's status-returning entry points: ``_launch(prof, info).<symbol>(...)``
raises WmdError naming the symbol that returned a failing status, and the profiler sees the call only when one is
installed."""
import pytest
import torch

from wavelet_monodepth_b200 import _lib, ops

WMD_ERR_SHAPE = -2                     # include/wmd.h


class _FakeLib:
    """Stands in for the loaded library: every entry point returns `rc` and records its name and arguments."""

    def __init__(self, rc):
        self.rc, self.calls = rc, []

    def wmd_status_string(self, rc):
        return b"unsupported size"

    def wmd_last_cuda_error(self):
        return 0

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name, args))
            return self.rc
        return call


def _no_events(*args, **kwargs):
    raise AssertionError("a CUDA event was created while no profiler is installed")


@pytest.mark.parametrize("prof", [None, "nchw_to_rows"])
def test_a_failing_call_names_the_symbol_it_called(monkeypatch, prof):
    fake = _FakeLib(WMD_ERR_SHAPE)
    monkeypatch.setattr(_lib, "_lib", fake)
    monkeypatch.setattr(ops, "_profiler", None)
    monkeypatch.setattr(torch.cuda, "Event", _no_events)
    infos = []
    with pytest.raises(_lib.WmdError, match=r"^wmd_nchw_to_rows_gated_amax_f32 failed: unsupported size \(status -2,"):
        ops._launch(prof, lambda: infos.append(1) or {}).wmd_nchw_to_rows_gated_amax_f32(1, None, 2.5)
    assert fake.calls == [("wmd_nchw_to_rows_gated_amax_f32", (1, None, 2.5))]
    assert infos == []                 # nothing was recorded


def test_a_successful_call_returns_quietly(monkeypatch):
    fake = _FakeLib(0)
    monkeypatch.setattr(_lib, "_lib", fake)
    monkeypatch.setattr(ops, "_profiler", None)
    monkeypatch.setattr(torch.cuda, "Event", _no_events)
    assert ops._launch("gate_map", dict).wmd_gate_map(7) is None
    assert fake.calls == [("wmd_gate_map", (7,))]


def _nchw_to_rows_gated_amax():
    x = torch.randn(1, 8, 4, 4, device="cuda")
    gate = torch.ones(1, 1, 4, 4, dtype=torch.uint8, device="cuda")
    amax = torch.zeros(1, device="cuda")
    return lambda: ops.nchw_to_rows(x, ld=4, gate=gate, amax=amax)          # ld < C


def _gather_rows_list_amax():
    x = torch.randn(1, 8, 4, 4, device="cuda")
    pixels = torch.arange(16, dtype=torch.int32, device="cuda")
    count = torch.tensor([16], dtype=torch.int32, device="cuda")
    amax = torch.zeros(1, device="cuda")
    return lambda: ops.gather_rows_list(x, pixels, count, ld=4, amax=amax)  # ld < C


def _conv_rows_tc():
    wp = ops.pack_weight(torch.randn(32, 128, 1, 1, device="cuda"), kind="tc")
    x0 = torch.randn(16, 128, device="cuda")
    return lambda: ops.conv_rows(x0, 128, wp, None, 32, 1, 4, 4, taps=1, pad=7)  # no such pad mode


@pytest.mark.gpu
@pytest.mark.parametrize("symbol, make", [("wmd_nchw_to_rows_gated_amax_f32", _nchw_to_rows_gated_amax),
                                          ("wmd_gather_rows_list_amax_f32", _gather_rows_list_amax),
                                          ("wmd_conv_rows_tc_splitk_f32", _conv_rows_tc)])
def test_a_rejected_call_names_its_entry_point(symbol, make):
    """Arguments the entry point rejects before it launches anything: the error names that entry point."""
    call = make()
    torch.cuda.synchronize()
    before = _lib.launch_count()
    with pytest.raises(_lib.WmdError, match=r"^%s failed: " % symbol):
        call()
    assert _lib.launch_count() == before
