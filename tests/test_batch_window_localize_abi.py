"""The ctypes record of pvio_b200_batch_window_localize has the header's LP64 layout (no GPU needed)."""
import ctypes as C

from pvio_b200 import _lib


def test_localize_record_matches_the_header():
    assert C.sizeof(_lib.CWindowLocalize) == 120                       # include/pvio_b200.h: 120 bytes on LP64
    assert _lib.CWindowLocalize.n_obs.offset == 24 and _lib.CWindowLocalize.n_new.offset == 64
    assert _lib.CWindowLocalize.summary.offset == 112
    assert "pvio_b200_batch_window_localize" in _lib.EXPORTS
