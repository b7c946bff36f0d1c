"""Argument validation of the two 3DGS-MCMC entry points without a GPU: every bad argument is rejected before any CUDA call,
and n = 0 is a no-op."""
import ctypes
import os

import pytest


@pytest.fixture(scope="module")
def L():
    from b200gs import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.lib()


D16, D8 = ctypes.c_void_p(16), ctypes.c_void_p(8)   # non-NULL dummies, 16- and 8-byte aligned; never dereferenced here


def test_relocation_rejects_bad_arguments(L):
    assert L.b200gs_mcmc_relocation(-1, D16, D16, D16, D16, 51, D16, D16, None) == -1
    assert b"n < 0" in L.b200gs_last_error()
    for k in range(6):
        args = [D16] * 6
        args[k] = None
        assert L.b200gs_mcmc_relocation(5, *args[:4], 51, *args[4:], None) == -1
        assert b"NULL" in L.b200gs_last_error()
    for n_max in (0, -3):
        assert L.b200gs_mcmc_relocation(5, D16, D16, D16, D16, n_max, D16, D16, None) == -1
        assert b"n_max" in L.b200gs_last_error()
    assert L.b200gs_mcmc_relocation(0, None, None, None, None, 51, None, None, None) == 0


def test_position_noise_rejects_bad_arguments(L):
    assert L.b200gs_mcmc_position_noise(-1, D16, D16, D16, D16, 1.0, 1, 0, None) == -1
    assert b"n < 0" in L.b200gs_last_error()
    for k in range(4):
        args = [D16] * 4
        args[k] = None
        assert L.b200gs_mcmc_position_noise(5, *args, 1.0, 1, 0, None) == -1
        assert b"NULL" in L.b200gs_last_error()
    assert L.b200gs_mcmc_position_noise(5, D16, D16, D8, D16, 1.0, 1, 0, None) == -1
    assert b"aligned" in L.b200gs_last_error()
    assert L.b200gs_mcmc_position_noise(0, None, None, None, None, 1.0, 2 ** 64 - 1, 2 ** 64 - 1, None) == 0
