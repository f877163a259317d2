"""Deterministic mode without a GPU: the C entry points are exported and bound, and every native call passes torch's
`are_deterministic_algorithms_enabled()` to its handle (a stand-in library records the calls)."""
import ctypes as C

import torch

from diamond_b200 import _lib, utils


def test_set_deterministic_entry_points_are_exported_and_bound():
    lib = _lib.lib()
    for pre in ("dmd_denoiser_", "dmd_rew_end_", "dmd_actor_critic_"):
        name = pre + "set_deterministic"
        assert _lib.SIGNATURES[name] == (C.c_int, [C.c_void_p, C.c_int])
        assert getattr(lib, name).restype is C.c_int
    assert lib.dmd_denoiser_set_deterministic(None, 1) != 0   # a null handle is refused
    assert b"null handle" in lib.dmd_last_error()


class _RecordingLib:
    def __init__(self):
        self.calls = []

    def dmd_x_create(self, cfg):
        return 1

    def dmd_x_num_tensors(self, h):
        return 1

    def dmd_x_packed_bytes(self, h):
        return 16

    def dmd_x_set_weights(self, h, arr, n, packed, stream):
        return 0

    def dmd_x_set_deterministic(self, h, on):
        self.calls.append(on)
        return 0


class _Module(utils.NativeStateMixin, torch.nn.Module):
    _NATIVE_PREFIX = "dmd_x_"

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(4))

    device = torch.device("cuda", 0)

    def _native_config(self):
        return C.c_int(0)

    def _state_tensors(self):
        return [self.w]

    def require_current_device(self, dev):
        pass

    def __del__(self):
        pass


def test_every_native_call_passes_torchs_flag(monkeypatch):
    fake = _RecordingLib()
    monkeypatch.setattr(utils._lib, "lib", lambda: fake)
    monkeypatch.setattr(utils._lib, "current_stream", lambda: None)
    monkeypatch.setattr(torch.Tensor, "data_ptr", lambda self: 0)
    monkeypatch.setattr(torch, "empty", lambda *a, **k: torch.zeros(16, dtype=torch.uint8))
    m = _Module()
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        m._native()
        torch.use_deterministic_algorithms(True)
        m._native()
        torch.use_deterministic_algorithms(True, warn_only=True)
        m._native()
        torch.use_deterministic_algorithms(False)
        m._native()
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)
    assert fake.calls == [0, 1, 1, 0]
