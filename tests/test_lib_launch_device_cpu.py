"""The launch device guard of `_lib.call`, without a GPU or the library: torch's device functions are replaced by a fake with a current-device
index, and the library by a recorder of (entry point, current device) per call.  A stream from `launch_stream(device)` carries its device, so
every call made with it runs with that device current, however many calls share the stream and whatever ran before."""
import contextlib
import ctypes
import re
import types

import pytest
import torch

from makani_b200 import _lib, sht


class _FakeCuda:
    def __init__(self):
        self.current = 0
        self.switches = 0
        self.calls = []     # (entry point, current device during the call)

    def __getattr__(self, name):       # the library: every entry point records the current device and succeeds
        if not name.startswith("b200sht_"):
            raise AttributeError(name)

        def entry(*args):
            self.calls.append((name, self.current))
            return 0
        return entry

    def index(self, dev):
        i = torch.device(dev).index if dev is not None else None
        return self.current if i is None else i

    @contextlib.contextmanager
    def device(self, index):
        old, self.current = self.current, index
        self.switches += 1
        try:
            yield
        finally:
            self.current = old


@pytest.fixture
def fake(monkeypatch):
    f = _FakeCuda()
    monkeypatch.setattr(torch.cuda, "current_device", lambda: f.current)
    monkeypatch.setattr(torch.cuda, "device", f.device)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: types.SimpleNamespace(cuda_stream=1000 + f.index(dev)))
    monkeypatch.setattr(_lib, "load", lambda: f)
    return f


CUDA0, CUDA1 = torch.device("cuda", 0), torch.device("cuda", 1)


def test_every_call_on_a_shared_stream_runs_on_its_device(fake):
    st = _lib.launch_stream(CUDA1)
    after = []
    for name in ("b200sht_a", "b200sht_b", "b200sht_c"):
        _lib.call(name, 7, st)
        after.append(fake.current)
    assert fake.calls == [("b200sht_a", 1), ("b200sht_b", 1), ("b200sht_c", 1)]
    assert after == [0, 0, 0]


def test_a_calls_device_does_not_depend_on_earlier_calls(fake):
    st0 = _lib.launch_stream(CUDA0)
    st1 = _lib.launch_stream(CUDA1)          # fetched after st0, used after st0's calls
    _lib.call("b200sht_first_on_0", st0)
    plan = sht.Plan(9, 16, 8, 9, "equiangular", True, CUDA1)     # a plan created for cuda:1 in between
    _lib.launch_stream(CUDA1)                                     # a stream fetched and never passed to call
    _lib.call("b200sht_second_on_0", st0)
    _lib.call("b200sht_on_1", st1)
    del plan
    assert fake.calls[0] == ("b200sht_first_on_0", 0)
    assert ("b200sht_plan_create_ex", 1) in fake.calls
    assert fake.calls[-2:] == [("b200sht_second_on_0", 0), ("b200sht_on_1", 1)]
    assert fake.current == 0


def test_plain_void_pointer_stream_is_not_switched(fake):
    _lib.launch_stream(CUDA1)
    _lib.call("b200sht_plain", ctypes.c_void_p(1234))
    _lib.call("b200sht_no_stream", 3)
    assert fake.calls == [("b200sht_plain", 0), ("b200sht_no_stream", 0)]
    assert fake.switches == 0


def test_current_device_stream_is_not_switched(fake):
    _lib.call("b200sht_x", _lib.launch_stream(CUDA0))
    _lib.call("b200sht_y", _lib.launch_stream("cuda"))
    assert fake.calls == [("b200sht_x", 0), ("b200sht_y", 0)]
    assert fake.switches == 0


def test_stream_is_the_last_parameter_of_every_entry_point():
    """`call` finds the device in args[-1], so every entry point of include/b200sht.h that takes a stream takes it last."""
    with open(_lib.HEADER_PATH) as f:
        text = re.sub(r"/\*.*?\*/|//[^\n]*", "", f.read(), flags=re.S)
    decls = re.findall(r"\b(b200sht_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", text)
    assert len(decls) >= 60
    with_stream = 0
    for name, params in decls:
        names = [re.findall(r"\w+", p)[-1] for p in params.split(",") if p.strip() and p.strip() != "void"]
        if "stream" in names:
            with_stream += 1
            assert names[-1] == "stream", name
            if name in _lib._SIGNATURES:
                assert _lib._SIGNATURES[name][1][-1] is ctypes.c_void_p, name
    assert with_stream >= 50


def test_dtype_code():
    assert _lib.dtype_code(torch.float32) == _lib.F32
    assert _lib.dtype_code(torch.bfloat16) == _lib.BF16
    with pytest.raises(_lib.B200ShtError):
        _lib.dtype_code(torch.float16)


def test_one_definition_of_each_helper():
    """the helpers sht re-exports (imported from there by benchmarks and scripts) are the _lib definitions"""
    assert sht._ptr is _lib.ptr and sht._stream is _lib.launch_stream and sht._dtype_code is _lib.dtype_code and sht._VP is ctypes.c_void_p
    t = torch.zeros(2)
    assert _lib.ptr(t).value == t.data_ptr() and _lib.ptr(None).value is None
