"""The device probe of the GLSL layer (tests/gpu_probe/glsl_probe.cu): compiled with the NVRTC library the product loads and
the options of the product's scene programs, loaded through the driver API in torch's current context.  No nvcc at test time.
"""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PROBE_SRC = os.path.join(ROOT, "tests", "gpu_probe", "glsl_probe.cu")
DEVICE_DIR = os.path.join(ROOT, "portal_b200", "csrc", "device")

# compile_cubin's option list (portal_b200/csrc/pe_program.cpp); tests/test_elementary_host.py pins the two together
OPTIONS = ["--gpu-architecture=sm_90a", "--std=c++20", "-default-device", "--fmad=false",
           "--prec-div=true", "--prec-sqrt=true", "--ftz=false"]

# function ids of pe_probe_f / pe_probe_f2
FUNCS = ["sin", "cos", "tan", "asin", "acos", "atan", "exp2", "exp", "log2", "log", "sinh", "cosh", "tanh", "sqrt", "inversesqrt"]
FUNCS2 = ["pow", "atan2", "mod"]
STAT_FIELDS = ["max_ulp", "max_abs", "n", "nonfinite_bad", "finite_bad", "special_bad"]


def nvrtc_library():
    """The NVRTC the product loads: $PORTAL_B200_NVRTC, else the toolkit's (PE_NVRTC_PATH in portal_b200/build.py)."""
    env = os.environ.get("PORTAL_B200_NVRTC")
    if env:
        return env
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    return os.path.join(cuda, "lib64", "libnvrtc.so.12")


def compile_probe(options=None, include_dir=None, source=PROBE_SRC, extra=(), want_log=False):
    """A probe source (glsl_probe.cu by default) -> sm_90a cubin bytes (options: OPTIONS; include_dir: the product's device
    headers; extra: further options of this probe, such as its own include directory or a -D).  want_log: return
    (cubin, NVRTC's log) instead."""
    nv = C.CDLL(nvrtc_library())
    with open(source, "rb") as f:
        src = f.read()
    prog = C.c_void_p()
    assert nv.nvrtcCreateProgram(C.byref(prog), src, os.path.basename(source).encode(), 0, None, None) == 0
    opts = [o.encode() for o in (OPTIONS if options is None else options)] + [b"--include-path=" + (include_dir or DEVICE_DIR).encode()]
    opts += [o.encode() for o in extra]
    arr = (C.c_char_p * len(opts))(*opts)
    rc = nv.nvrtcCompileProgram(prog, len(opts), arr)
    size = C.c_size_t()
    nv.nvrtcGetProgramLogSize(prog, C.byref(size))
    log = C.create_string_buffer(size.value)
    nv.nvrtcGetProgramLog(prog, log)
    try:
        assert rc == 0, log.value.decode(errors="replace")[-4000:]
        nv.nvrtcGetCUBINSize(prog, C.byref(size))
        cubin = C.create_string_buffer(size.value)
        assert nv.nvrtcGetCUBIN(prog, cubin) == 0
        return (cubin.raw, log.value.decode(errors="replace")) if want_log else cubin.raw
    finally:
        nv.nvrtcDestroyProgram(C.byref(prog))


class Probe:
    """The probe's kernels, launched on torch's current stream of cuda:0."""

    def __init__(self, torch, options=None, include_dir=None, source=PROBE_SRC, extra=(),
                 kernels=("accuracy_unary", "accuracy_binary", "eval_unary", "eval_binary")):
        self.torch = torch
        torch.cuda.init()
        torch.empty(1, device="cuda")                         # makes torch's primary context current on this thread
        self.cu = C.CDLL("libcuda.so.1")
        self._cubin = compile_probe(options, include_dir, source, extra)
        self.mod = C.c_void_p()
        self._check(self.cu.cuModuleLoadData(C.byref(self.mod), self._cubin))
        self.fns = {}
        for name in kernels:
            f = C.c_void_p()
            self._check(self.cu.cuModuleGetFunction(C.byref(f), self.mod, name.encode()))
            self.fns[name] = f

    def _check(self, rc):
        assert rc == 0, f"CUDA driver error {rc}"

    def close(self):
        self.torch.cuda.synchronize()
        self._check(self.cu.cuModuleUnload(self.mod))

    def _launch(self, name, grid, block, args):
        holders = [a for a in args]
        ptrs = (C.c_void_p * len(holders))(*[C.cast(C.pointer(h), C.c_void_p) for h in holders])
        stream = C.c_void_p(self.torch.cuda.current_stream().cuda_stream)
        self._check(self.cu.cuLaunchKernel(self.fns[name], grid, 1, 1, block, 1, 1, 0, stream, ptrs, None))

    def _dev(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def _stats(self, t):
        raw = t.cpu().numpy()
        out = []
        for row in raw:
            d = dict(zip(STAT_FIELDS, (int(v) for v in row)))
            d["max_ulp"] = float(np.array([row[0]], np.uint64).view(np.float64)[0])
            d["max_abs"] = float(np.array([row[1]], np.uint64).view(np.float64)[0])
            out.append(d)
        return out

    def accuracy_unary(self, fn, bands, first=0, count=1 << 32):
        """Per band (lo, hi) of |x|: worst ulp / absolute error against the double-precision function, and bad special values,
        over the input bit patterns first .. first + count - 1 (all 2^32 by default)."""
        lo = self._dev(np.array([b[0] for b in bands], np.float32))
        hi = self._dev(np.array([b[1] for b in bands], np.float32))
        st = self.torch.zeros((len(bands), len(STAT_FIELDS)), dtype=self.torch.int64, device="cuda")
        self._launch("accuracy_unary", 132 * 16, 256,
                     [C.c_int(FUNCS.index(fn)), C.c_ulonglong(first), C.c_ulonglong(count), C.c_int(len(bands)),
                      C.c_void_p(lo.data_ptr()), C.c_void_p(hi.data_ptr()), C.c_void_p(st.data_ptr())])
        self.torch.cuda.synchronize()
        return self._stats(st)

    def accuracy_binary(self, fn, xs, ys):
        """Worst ulp / absolute error over the grid xs x ys (pairs with a sub-normal exact result left out)."""
        dx, dy = self._dev(np.asarray(xs, np.float32)), self._dev(np.asarray(ys, np.float32))
        st = self.torch.zeros((1, len(STAT_FIELDS)), dtype=self.torch.int64, device="cuda")
        self._launch("accuracy_binary", 132 * 16, 256, [C.c_int(FUNCS2.index(fn)), C.c_void_p(dx.data_ptr()), C.c_uint(len(xs)),
                                                        C.c_void_p(dy.data_ptr()), C.c_uint(len(ys)), C.c_void_p(st.data_ptr())])
        self.torch.cuda.synchronize()
        return self._stats(st)[0]

    def eval_unary(self, fn, xs):
        x = self._dev(np.asarray(xs, np.float32))
        out = self.torch.empty_like(x)
        n = x.numel()
        self._launch("eval_unary", (n + 255) // 256, 256, [C.c_int(FUNCS.index(fn)), C.c_void_p(x.data_ptr()),
                                                           C.c_void_p(out.data_ptr()), C.c_uint(n)])
        return out.cpu().numpy()

    def eval_binary(self, fn, xs, ys):
        x, y = self._dev(np.asarray(xs, np.float32)), self._dev(np.asarray(ys, np.float32))
        out = self.torch.empty_like(x)
        n = x.numel()
        self._launch("eval_binary", (n + 255) // 256, 256, [C.c_int(FUNCS2.index(fn)), C.c_void_p(x.data_ptr()),
                                                            C.c_void_p(y.data_ptr()), C.c_void_p(out.data_ptr()), C.c_uint(n)])
        return out.cpu().numpy()
