"""ctypes binding of include/cmixb200.h.

`Predictor` mirrors the reference's `class Predictor` (reference src/predictor.h:17-53):
Predict() / Perceive(bit) / Pretrain(bit), plus the bulk compress-direction call the
reference's Compress() loop (src/runner.cpp:101-119) maps to.
"""
import ctypes
import os
import subprocess

import numpy as np

N_EXT = 2022
_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
PRODUCT_LIB = os.path.join(CSRC, "libcmixb200.so")
LIB_PATH = os.environ.get("CMIXB200_LIB") or PRODUCT_LIB   # CMIXB200_LIB: load a variant (profiling, jitter, census) instead
UNITS = ["engine.cu", "fxcm_dev.cu", "paq8_dev.cu"]         # the three device programs, compiled side by side
NVCC_COMPILE = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]
NVCC_LINK = ["-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC"]

_lib = None


def build_library(force=False, defines=(), out_dir=None):
    """Compile the UNITS for sm_90a and link them into libcmixb200.so; rebuilds when a source is newer. Returns its path.

    By default this is the product, in csrc/. A variant (e.g. defines=["-DCMIXB200_JITTER"]) is built into its own out_dir."""
    assert not defines or out_dir, "a variant build needs an out_dir of its own"
    out_dir = out_dir or CSRC
    lib, objs = os.path.join(out_dir, "libcmixb200.so"), [os.path.join(out_dir, u[:-3] + ".o") for u in UNITS]
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))]
    srcs.append(os.path.join(os.path.dirname(_HERE), "include", "cmixb200.h"))
    if not force and os.path.exists(lib) and all(os.path.getmtime(lib) >= os.path.getmtime(s) for s in srcs):
        return lib
    jobs = [subprocess.Popen(["nvcc"] + NVCC_COMPILE + list(defines) + ["-c", os.path.join(CSRC, u), "-o", obj])
            for u, obj in zip(UNITS, objs)
            if force or not os.path.exists(obj) or any(os.path.getmtime(obj) < os.path.getmtime(s) for s in srcs)]
    if any(j.wait() != 0 for j in jobs):
        raise RuntimeError("cmix_b200: nvcc failed")
    subprocess.run(["nvcc"] + NVCC_LINK + objs + ["-o", lib], check=True)
    return lib


def load_library():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("cmix_b200: %s is missing - run __graft_entry__.build() (nvcc, sm_90a); "
                           "there is no CPU fallback" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    c = ctypes
    vp = c.c_void_p
    lib.cmixb200_create.argtypes = [vp, c.c_char_p, c.c_int, c.POINTER(vp)]
    lib.cmixb200_create.restype = c.c_int
    lib.cmixb200_create_ex.argtypes = [vp, c.c_char_p, c.c_int, c.c_uint, c.POINTER(vp)]
    lib.cmixb200_create_ex.restype = c.c_int
    lib.cmixb200_destroy.argtypes = [vp]
    lib.cmixb200_destroy.restype = None
    lib.cmixb200_predict.argtypes = [vp]
    lib.cmixb200_predict.restype = c.c_float
    lib.cmixb200_perceive.argtypes = [vp, c.c_int]
    lib.cmixb200_pretrain.argtypes = [vp, c.c_int]
    lib.cmixb200_feed_external_bit.argtypes = [vp, vp]
    lib.cmixb200_feed_external_byte.argtypes = [vp, vp]
    lib.cmixb200_code_bytes.argtypes = [vp, vp, c.c_size_t, vp, vp, vp]
    lib.cmixb200_code_bytes_device.argtypes = [vp, vp, c.c_size_t, vp, vp, vp]
    lib.cmixb200_code_batch_device.argtypes = [vp, c.c_int, vp, c.c_size_t, vp, vp, vp]
    lib.cmixb200_code_batch.argtypes = [vp, c.c_int, vp, c.c_size_t, vp, vp, vp]
    lib.cmixb200_coder_begin.argtypes = [vp, c.c_size_t]
    lib.cmixb200_coder_finish.argtypes = [vp, vp, c.c_size_t, c.POINTER(c.c_size_t)]
    lib.cmixb200_pretrain_bytes.argtypes = [vp, vp, c.c_size_t]
    lib.cmixb200_decode_bytes.argtypes = [vp, vp, c.c_size_t, vp, c.c_size_t]
    lib.cmixb200_last_error.restype = c.c_char_p
    lib.cmixb200_kernel_launches.argtypes = [vp]
    lib.cmixb200_kernel_launches.restype = c.c_ulonglong
    lib.cmixb200_time_mix_kernel.argtypes = [vp, c.c_int]
    lib.cmixb200_time_mix_kernel.restype = None
    lib.cmixb200_kernel_ms.argtypes = [vp, c.c_int, c.POINTER(c.c_ulonglong)]
    lib.cmixb200_kernel_ms.restype = c.c_double
    lib.cmixb200_mix_stream.argtypes = [vp]
    lib.cmixb200_mix_stream.restype = vp
    lib.cmixb200_debug_fetch.argtypes = [vp, c.c_int, vp, c.c_size_t]
    _lib = lib
    return lib


def _check(lib, rc, what):
    if rc != 0:
        raise RuntimeError("cmix_b200.%s failed (%d): %s" % (what, rc, lib.cmixb200_last_error().decode()))


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return a.ctypes.data
    return a.data_ptr()  # torch tensor


class Predictor:
    """Mirror of the reference `Predictor` (src/predictor.h:17-53) on one GPU."""

    REPLAY = {"fxcm": 1, "paq8": 2}

    def __init__(self, vocab, dictionary_path=None, device=0, replay=()):
        """`replay`: model groups ("fxcm", "paq8") whose outputs are replayed instead of computed on the device."""
        self._lib = load_library()
        v = np.ascontiguousarray(np.asarray(vocab, dtype=np.uint8))
        assert v.size == 256
        h = ctypes.c_void_p()
        d = dictionary_path.encode() if dictionary_path else None
        mask = 0
        for name in replay:
            mask |= self.REPLAY[name]
        _check(self._lib, self._lib.cmixb200_create_ex(v.ctypes.data, d, int(device), mask, ctypes.byref(h)), "create")
        self._h = h
        self.device = device

    def close(self):
        if getattr(self, "_h", None):
            self._lib.cmixb200_destroy(self._h)
            self._h = None

    __del__ = close

    # --- the reference surface -------------------------------------------------
    def Predict(self):
        p = self._lib.cmixb200_predict(self._h)
        if p < 0:
            raise RuntimeError("cmix_b200.predict failed: %s" % self._lib.cmixb200_last_error().decode())
        return p

    def Perceive(self, bit):
        _check(self._lib, self._lib.cmixb200_perceive(self._h, int(bit)), "perceive")

    def Pretrain(self, bit):
        _check(self._lib, self._lib.cmixb200_pretrain(self._h, int(bit)), "pretrain")

    # --- replayed model streams ------------------------------------------------
    def feed_external_bit(self, codes):
        codes = np.ascontiguousarray(codes, dtype=np.uint16)
        assert codes.size == N_EXT
        _check(self._lib, self._lib.cmixb200_feed_external_bit(self._h, codes.ctypes.data), "feed_external_bit")

    def feed_external_byte(self, ppmd):
        ppmd = np.ascontiguousarray(ppmd, dtype=np.float32)
        assert ppmd.size == 256
        _check(self._lib, self._lib.cmixb200_feed_external_byte(self._h, ppmd.ctypes.data), "feed_external_byte")

    # --- bulk paths --------------------------------------------------------------
    def code_bytes(self, data, ext=None, ppmd=None):
        """Host buffers in, host probabilities out (one float per bit)."""
        data = np.ascontiguousarray(np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else data)
        n = data.size
        if ext is not None:
            ext = np.ascontiguousarray(ext, dtype=np.uint16)
            assert ext.size == n * 8 * N_EXT
        if ppmd is not None:
            ppmd = np.ascontiguousarray(ppmd, dtype=np.float32)
            assert ppmd.size == n * 256
        out = np.empty(n * 8, dtype=np.float32)
        _check(self._lib, self._lib.cmixb200_code_bytes(self._h, _ptr(data), n, _ptr(ext), _ptr(ppmd), _ptr(out)), "code_bytes")
        return out

    def code_bytes_device(self, d_bytes, n_bytes, d_ext, d_ppmd, d_p_out):
        """All arguments are torch CUDA tensors (or None) already resident in HBM."""
        _check(self._lib, self._lib.cmixb200_code_bytes_device(self._h, _ptr(d_bytes), n_bytes, _ptr(d_ext), _ptr(d_ppmd),
                                                                _ptr(d_p_out)), "code_bytes_device")

    def coder_begin(self, capacity_bytes):
        """Start the device arithmetic coder (Encoder, src/coder/encoder.cpp): bulk calls now also emit archive bytes."""
        _check(self._lib, self._lib.cmixb200_coder_begin(self._h, int(capacity_bytes)), "coder_begin")
        self._coder_cap = int(capacity_bytes)

    def coder_finish(self):
        """Encoder::Flush; returns the archive bytes (no runner.cpp header)."""
        out = np.empty(self._coder_cap, dtype=np.uint8)
        n = ctypes.c_size_t(0)
        _check(self._lib, self._lib.cmixb200_coder_finish(self._h, out.ctypes.data, out.size, ctypes.byref(n)), "coder_finish")
        return out[:n.value].tobytes()

    def decode_bytes(self, archive, n_bytes):
        """Decoder::Decode on the device: n_bytes of the stream from the arithmetic-coded archive body."""
        arch = np.ascontiguousarray(np.frombuffer(bytes(archive), dtype=np.uint8))
        out = np.empty(int(n_bytes), dtype=np.uint8)
        _check(self._lib, self._lib.cmixb200_decode_bytes(self._h, arch.ctypes.data, arch.size, out.ctypes.data, out.size), "decode_bytes")
        return out

    def pretrain_bytes(self, data):
        data = np.ascontiguousarray(np.frombuffer(bytes(data), dtype=np.uint8))
        _check(self._lib, self._lib.cmixb200_pretrain_bytes(self._h, data.ctypes.data, data.size), "pretrain_bytes")

    @property
    def kernel_launches(self):
        return int(self._lib.cmixb200_kernel_launches(self._h))

    def time_mix_kernel(self, enable=True):
        self._lib.cmixb200_time_mix_kernel(self._h, 1 if enable else 0)

    def kernel_ms(self, which):
        """(total ms, launches) of one bulk kernel since time_mix_kernel(True): 0 mix, 1 small, 2 lstm, 3 ppmd, 4 fxcm, 5 paq8."""
        n = ctypes.c_ulonglong(0)
        ms = self._lib.cmixb200_kernel_ms(self._h, int(which), ctypes.byref(n))
        return float(ms), int(n.value)

    @property
    def mix_stream(self):
        return int(self._lib.cmixb200_mix_stream(self._h) or 0)

    def debug_fetch(self, what, shape, dtype):
        out = np.empty(shape, dtype=dtype)
        _check(self._lib, self._lib.cmixb200_debug_fetch(self._h, what, out.ctypes.data, out.nbytes), "debug_fetch")
        return out


def code_batch_device(preds, d_bytes, n_bytes, d_ext, d_ppmd, d_p_out):
    """Advance len(preds) independent predictors by n_bytes each in one launch set."""
    lib = load_library()
    n = len(preds)
    VP = ctypes.c_void_p * n
    hs = VP(*[p._h.value for p in preds])
    by = VP(*[_ptr(t) for t in d_bytes])
    ex = VP(*[_ptr(t) for t in d_ext]) if d_ext is not None else None
    pp = VP(*[_ptr(t) for t in d_ppmd]) if d_ppmd is not None else None
    po = VP(*[_ptr(t) for t in d_p_out])
    _check(lib, lib.cmixb200_code_batch_device(hs, n, by, n_bytes, ex, pp, po), "code_batch_device")


def code_batch(preds, bytes_, n_bytes, ext, ppmd, p_out):
    """Host-buffer twin of code_batch_device: numpy arrays or pinned CPU torch tensors, one per predictor.

    Inputs are staged to the device in double-buffered sub-steps inside the call; p_out[s] (float32,
    n_bytes*8) receives what Predict() returned before each bit.
    """
    lib = load_library()
    n = len(preds)
    VP = ctypes.c_void_p * n
    hs = VP(*[p._h.value for p in preds])
    by = VP(*[_ptr(t) for t in bytes_])
    ex = VP(*[_ptr(t) for t in ext]) if ext is not None else None
    pp = VP(*[_ptr(t) for t in ppmd]) if ppmd is not None else None
    po = VP(*[_ptr(t) for t in p_out])
    _check(lib, lib.cmixb200_code_batch(hs, n, by, n_bytes, ex, pp, po), "code_batch")
