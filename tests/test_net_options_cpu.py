"""CPU: ctpn_net_set_option of the test library, which needs no device."""
import ctypes as C
import os

from ctpn_b200 import _native as N

# the test library next to the tests of the tree the package was loaded from (as _native.py finds it for CTPN_B200_LIB=dbg)
DBG_LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(N.__file__)))), "tests", "_native",
                       "libctpn_b200_dbg.so")
ARITH_F16F8 = 4     # include/ctpn_b200.h


def test_simt_convolutions_are_refused_on_an_f16f8_net():
    """The SIMT reference kernels read bf16 planes only: "conv_simt" is refused on an F16F8 net, accepted on bf16x2."""
    dbg = C.CDLL(DBG_LIB)
    for mode, want in ((ARITH_F16F8, N.ERR_INVALID), (2, 0)):
        net = C.c_void_p()
        assert dbg.ctpn_net_create(C.byref(net), mode) == 0
        assert dbg.ctpn_net_set_option(net, b"conv_simt", 1) == want
        assert dbg.ctpn_net_set_option(net, b"conv_simt", 0) == 0
        dbg.ctpn_net_destroy(net)
