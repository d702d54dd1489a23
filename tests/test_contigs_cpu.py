"""CPU checks of the contig -> window entry points of the C ABI (gnm_contig_windows, gnm_gather_windows,
gnm_forward_windows): bad arguments fail with a message before any device work, so no GPU is needed."""
import ctypes as C

import pytest

from genomad_b200 import engine


@pytest.fixture(scope="module")
def lib():
    return engine.load_library()


def _fails(lib, rc, *words):
    assert rc != 0
    msg = lib.gnm_last_error().decode()
    for w in words:
        assert w in msg, msg


def test_contig_windows_rejects_bad_arguments(lib):
    nw = C.c_int64(-7)
    _fails(lib, lib.gnm_contig_windows(None, None, None, 1, 0, None, None, 0, None, C.byref(nw), None),
           "gnm_contig_windows", "null handle")
    fake = C.c_void_p(1)          # never dereferenced: the argument checks come first
    _fails(lib, lib.gnm_contig_windows(fake, None, None, -1, 0, None, None, 0, None, C.byref(nw), None),
           "gnm_contig_windows", "negative contig count")
    _fails(lib, lib.gnm_contig_windows(fake, None, None, 1, 0, None, None, -1, None, C.byref(nw), None),
           "gnm_contig_windows", "negative capacity")
    _fails(lib, lib.gnm_contig_windows(fake, None, None, 1, 0, None, None, 10, None, C.byref(nw), None),
           "gnm_contig_windows", "null buffer")
    _fails(lib, lib.gnm_contig_windows(fake, None, None, 0, 0, None, None, 0, None, None, None),
           "gnm_contig_windows", "null buffer")
    assert nw.value == -7         # nothing written on an argument error


@pytest.mark.parametrize("name", ["gnm_gather_windows", "gnm_forward_windows"])
def test_window_entry_points_reject_bad_arguments(lib, name):
    fn = getattr(lib, name)
    _fails(lib, fn(None, None, None, None, 4, None, None), name, "null handle")
    fake = C.c_void_p(1)
    _fails(lib, fn(fake, None, None, None, -1, None, None), name, "negative window count")
    _fails(lib, fn(fake, None, None, None, 4, None, None), name, "null buffer")
    assert fn(fake, None, None, None, 0, None, None) == 0      # nothing to do: no device work, no error
