"""Host-side validation of minigpt4_b200_session_copy and the state save / restore entry points: NULL contexts, NULL arrays and n outside
1..64 are refused before any context is looked at, so these run without a GPU."""
import ctypes

import pytest

N_MAX = 64


def _dsts(n=N_MAX + 1):
    return ctypes.cast((ctypes.c_void_p * n)(), ctypes.c_void_p)


@pytest.mark.parametrize("n", [0, -1, N_MAX + 1, 1, 3, N_MAX])
def test_session_copy_refuses_null_arguments(ext, n):
    assert ext.L.minigpt4_b200_session_copy(None, _dsts(), n) == 8          # FailedToAddString
    assert ext.L.minigpt4_b200_session_copy(None, None, n) == 8
    ms = ctypes.c_float(-1)
    assert ext.L.minigpt4_b200_session_copy_timed(None, _dsts(), n, ctypes.byref(ms)) == 8
    assert ms.value == -1


def test_state_entry_points_refuse_a_null_context(ext):
    assert ext.L.minigpt4_b200_state_size(None) == -1
    buf = (ctypes.c_uint8 * 256)()
    written = ctypes.c_longlong(-7)
    assert ext.L.minigpt4_b200_state_save(None, buf, 256, ctypes.byref(written)) == 8
    assert ext.L.minigpt4_b200_state_save(None, None, 0, None) == 8
    assert written.value == -7
    assert ext.L.minigpt4_b200_state_load(None, buf, 256) == 8
    assert ext.L.minigpt4_b200_state_load(None, None, 0) == 8


def test_new_symbols_are_declared(ext):
    import minigpt4_cpp_b200.minigpt4_library as ml
    for sym in ("minigpt4_b200_session_copy", "minigpt4_b200_session_copy_timed", "minigpt4_b200_state_size", "minigpt4_b200_state_save",
                "minigpt4_b200_state_load"):
        assert sym in ml.EXT_SYMBOLS
        assert hasattr(ext.L, sym)
    assert all(hasattr(ml.B200, m) for m in ("session_copy", "state_save", "state_load"))
