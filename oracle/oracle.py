"""ctypes wrapper over oracle/_build/liboracle.so (C restatement of the reference's `Network`,
the reference's Tests/FlashAttentionTests/Utilities/Network.swift:70-403).

TEST INFRASTRUCTURE: parity unpinned against reference-generated vectors (none exist; the
reference cannot run here) -- pinned instead by oracle_np.py (float64) + finite differences, see
tests/test_oracle.py.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liboracle.so")
_lib = None

FP32, FP16, BF16 = 0, 1, 2  # GEMMOperandPrecision raw values (GEMMOperandPrecision.swift:33-37)


def build(force=False):
    """Compile the C oracle (gcc only; no GPU, no reference sources copied)."""
    src = os.path.join(_HERE, "network_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_SO)
        fp = ctypes.POINTER(ctypes.c_float)
        i = ctypes.c_int
        _lib.oracle_network_init.argtypes = [i, i, i, ctypes.c_uint64, fp, fp, fp, fp]
        _lib.oracle_inference_attention.argtypes = [i, i, i, fp, fp, fp, fp, fp, i]
        _lib.oracle_d_terms.argtypes = [i, i, i, fp, fp, fp, fp, fp, i]
        for name in ("oracle_derivative_v", "oracle_derivative_k", "oracle_derivative_q"):
            getattr(_lib, name).argtypes = [i, i, i, fp, fp, fp, fp, fp, i]
        _lib.oracle_loss.argtypes = [i, i, i, fp, fp, fp, fp]
        _lib.oracle_loss.restype = ctypes.c_double
        _lib.oracle_encode.argtypes = [fp, ctypes.c_void_p, ctypes.c_size_t, i]
        _lib.oracle_decode.argtypes = [ctypes.c_void_p, fp, ctypes.c_size_t, i]
        _lib.oracle_max_threads.restype = i
    return _lib


def _fp(a):
    assert a.dtype == np.float32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def max_threads():
    return int(lib().oracle_max_threads())


class Network:
    """Mirror of the reference's `struct Network` (Network.swift:70-113): seeded Q, K, V, dO plus
    the oracle outputs. Arrays are row-major float32: Q,dO [R,D]; K,V [C,D]."""

    def __init__(self, rowDimension, columnDimension, headDimension, seed=0, threads=1):
        self.rowDimension, self.columnDimension, self.headDimension = (
            int(rowDimension), int(columnDimension), int(headDimension))
        R, C, D = self.rowDimension, self.columnDimension, self.headDimension
        self.threads = threads
        self.Q = np.empty((R, D), np.float32)
        self.K = np.empty((C, D), np.float32)
        self.V = np.empty((C, D), np.float32)
        self.dO = np.empty((R, D), np.float32)
        lib().oracle_network_init(R, C, D, seed, _fp(self.Q), _fp(self.K), _fp(self.V), _fp(self.dO))

    def round_inputs(self, precision_qkv, precision_dO=None):
        """Round Q,K,V (and dO) through a 16-bit memory format, exactly as the kernel sees them
        (MTLContext+Buffers.swift:31-44), so oracle and kernel consume identical values."""
        self.Q = roundtrip(self.Q, precision_qkv)
        self.K = roundtrip(self.K, precision_qkv)
        self.V = roundtrip(self.V, precision_qkv)
        self.dO = roundtrip(self.dO, precision_qkv if precision_dO is None else precision_dO)
        return self

    def _dims(self):
        return self.rowDimension, self.columnDimension, self.headDimension

    def inferenceAttention(self, with_L=False):
        R, C, D = self._dims()
        O = np.empty((R, D), np.float32)
        L = np.empty((R,), np.float32) if with_L else None
        lib().oracle_inference_attention(R, C, D, _fp(self.Q), _fp(self.K), _fp(self.V), _fp(O),
                                         _fp(L) if with_L else None, self.threads)
        return (O, L) if with_L else O

    def createLTerms(self):
        return self.inferenceAttention(with_L=True)[1]

    def createDTerms(self):
        R, C, D = self._dims()
        out = np.empty((R,), np.float32)
        lib().oracle_d_terms(R, C, D, _fp(self.Q), _fp(self.K), _fp(self.V), _fp(self.dO), _fp(out),
                             self.threads)
        return out

    def _deriv(self, fn, shape):
        R, C, D = self._dims()
        out = np.empty(shape, np.float32)
        fn(R, C, D, _fp(self.Q), _fp(self.K), _fp(self.V), _fp(self.dO), _fp(out), self.threads)
        return out

    def derivativeV(self):
        return self._deriv(lib().oracle_derivative_v, (self.columnDimension, self.headDimension))

    def derivativeK(self):
        return self._deriv(lib().oracle_derivative_k, (self.columnDimension, self.headDimension))

    def derivativeQ(self):
        return self._deriv(lib().oracle_derivative_q, (self.rowDimension, self.headDimension))

    def loss(self):
        R, C, D = self._dims()
        return float(lib().oracle_loss(R, C, D, _fp(self.Q), _fp(self.K), _fp(self.V), _fp(self.dO)))


def encode(array, precision):
    """float32 -> raw memory image in `precision` (FP16 = RNE, BF16 = truncate)."""
    a = np.ascontiguousarray(array, np.float32)
    if precision == FP32:
        return a.copy()
    out = np.empty(a.shape, np.uint16)
    lib().oracle_encode(_fp(a), out.ctypes.data_as(ctypes.c_void_p), a.size, precision)
    return out


def decode(raw, precision):
    if precision == FP32:
        return np.ascontiguousarray(raw, np.float32).copy()
    r = np.ascontiguousarray(raw, np.uint16)
    out = np.empty(r.shape, np.float32)
    lib().oracle_decode(r.ctypes.data_as(ctypes.c_void_p), _fp(out), r.size, precision)
    return out


def roundtrip(array, precision):
    return decode(encode(array, precision), precision)
