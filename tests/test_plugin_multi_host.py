"""The multi-GPU plugin's entry points on their argument checks (no GPU needed): a plugin over pm_multi needs a
pm_multi, and the version of no pm_multi is 0."""
import ctypes as C

from protocol_b200 import abi
from protocol_b200._lib import load


def test_create_multi_refuses_null():
    lib = load()
    pol = abi.PmPluginPolicy(1, 1, 1, 0)
    h = C.c_void_p()
    assert lib.pm_plugin_create_multi(None, C.byref(pol), C.byref(h)) == abi.PM_E_INVALID
    assert not h.value
    assert lib.pm_plugin_create_multi(None, None, C.byref(h)) == abi.PM_E_INVALID


def test_multi_table_version_of_null_is_zero():
    assert load().pm_multi_table_version(None) == 0
