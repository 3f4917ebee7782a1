"""ctypes binding of the C ABI declared in ``include/torchsde_b200.h``.

This is the only place where Python meets the CUDA library.  Tensors cross as raw device
pointers (``Tensor.data_ptr()``) plus sizes; the stream is torch's current CUDA stream, so every
launch is ordered with the surrounding torch ops and can be captured into a CUDA graph.

There is deliberately no fallback: if the shared library is missing, importing the solver
raises (`LibraryNotBuilt`) telling the user to run ``python __graft_entry__.py`` (build()).
"""
import ctypes
import importlib
import os

import torch

_LIB_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'lib')
# TORCHSDE_B200_LIB: load another build of the same ABI instead (A/B measurements of kernel changes on one box)
LIB_PATH = os.environ.get('TORCHSDE_B200_LIB') or os.path.join(_LIB_DIR, 'libtorchsde_b200.so')

F32, F64 = 0, 1
NOISE_DIAGONAL, NOISE_GENERAL = 0, 1
SRC_MEMORY, SRC_COUNTER, SRC_UNIT = 0, 1, 2
EINVAL = -22
ECOMPILE = -38  # TSDE_ECOMPILE: an element-wise program could not be compiled (NVRTC missing, or its log)
FLAG_G_BROADCAST = 1
LOGQP_GENERAL_MAX = 16384  # TSDE_LOGQP_GENERAL_MAX


def logqp_general_fits(d, m):
    """Whether tsde_logqp_augment takes a general-noise (d, m) row: its min(d,m) x max(d,m) matrix plus f - h within
    LOGQP_GENERAL_MAX elements of shared memory."""
    return min(d, m) * max(d, m) + d <= LOGQP_GENERAL_MAX


def _program_launch(dtype):
    # (a one-row diagonal launch: what tsde_pointwise_source / _compile read of it is the dtype)
    return Launch(dtype_code(dtype), NOISE_DIAGONAL, 1, 4, 4, None)


def pointwise_source(prog, dtype):
    """The CUDA source the library compiles for Milstein program `prog` (a Pointwise) in `dtype`, or None if the library
    refuses the program (tsde_pointwise_source; no device needed)."""
    L = _program_launch(dtype)
    n = lib().tsde_pointwise_source(ctypes.byref(L), ctypes.byref(prog), None, 0)
    if n < 0:
        return None
    buf = ctypes.create_string_buffer(n + 1)
    lib().tsde_pointwise_source(ctypes.byref(L), ctypes.byref(prog), buf, n + 1)
    return buf.value.decode()


def compile_pointwise(prog, dtype):
    """tsde_pointwise_compile: compile and load the kernels of Milstein program `prog` in `dtype`; 0 or an error
    code."""
    return lib().tsde_pointwise_compile(ctypes.byref(_program_launch(dtype)), ctypes.byref(prog))


def _general_launch(dtype, d, m):
    # (a one-row general launch: what tsde_pointwise_source / _compile read of it is the dtype, d and m)
    return Launch(dtype_code(dtype), NOISE_GENERAL, 1, d, m, None)


def general_pointwise_source(prog, dtype, d, m):
    """The CUDA source the library compiles for general-noise program `prog` in `dtype` with m Brownian channels, or None
    if the library refuses the program (tsde_pointwise_source on a GENERAL launch; no device needed)."""
    L = _general_launch(dtype, d, m)
    n = lib().tsde_pointwise_source(ctypes.byref(L), ctypes.byref(prog), None, 0)
    if n < 0:
        return None
    buf = ctypes.create_string_buffer(n + 1)
    lib().tsde_pointwise_source(ctypes.byref(L), ctypes.byref(prog), buf, n + 1)
    return buf.value.decode()


def compile_general_pointwise(prog, dtype, d, m):
    """tsde_pointwise_compile on a GENERAL launch: compile and load the Euler and midpoint kernels of general-noise
    program `prog` (the sra1, Euler-Heun or reversible-Heun kernels if it is tagged PW_LAYOUT_GENERAL_SRA, _EULER_HEUN
    or _REVERSIBLE_HEUN); 0 or an error code."""
    return lib().tsde_pointwise_compile(ctypes.byref(_general_launch(dtype, d, m)), ctypes.byref(prog))


def compile_adaptive_pointwise(prog, dtype):
    """tsde_adaptive_pointwise_compile: compile and load the adaptive proposal kernel of Milstein program `prog` in
    `dtype`; 0 or an error code."""
    return lib().tsde_adaptive_pointwise_compile(ctypes.byref(_program_launch(dtype)), ctypes.byref(prog))


class LibraryNotBuilt(RuntimeError):
    pass


class Launch(ctypes.Structure):
    _fields_ = [('dtype', ctypes.c_int32), ('noise_type', ctypes.c_int32), ('rows', ctypes.c_int64),
                ('d', ctypes.c_int64), ('m', ctypes.c_int64), ('stream', ctypes.c_void_p)]


class Noise(ctypes.Structure):
    _fields_ = [('source', ctypes.c_int32), ('want_u', ctypes.c_int32), ('w', ctypes.c_void_p),
                ('u', ctypes.c_void_p), ('key', ctypes.c_void_p), ('cell_id', ctypes.c_uint64),
                ('row_offset', ctypes.c_int64), ('n_cells', ctypes.c_int32), ('flags', ctypes.c_int32),
                ('h', ctypes.c_double), ('cell_h', ctypes.c_void_p), ('h_total', ctypes.c_double)]


PW_MAX_INSTR, PW_MAX_OPERANDS, PW_MAX_REGS = 96, 24, 24  # TSDE_PW_MAX_*
PW_SRC_Y, PW_SRC_GO, PW_OPERAND0 = 0xFE, 0xFF, 0x80
PW_MUL, PW_ADD, PW_SUB, PW_DIV, PW_NEG, PW_SQRT = range(6)
PW_LT, PW_LE, PW_EQ, PW_MAXIMUM, PW_MINIMUM, PW_ABS, PW_SEL = range(8, 15)  # (6, 7 reserved)
# the transcendental ops, which only the compiled layouts run (15 reserved)
(PW_EXP, PW_LOG, PW_SIN, PW_COS, PW_TANH, PW_LOG1P, PW_EXPM1, PW_RSQRT, PW_SIGMOID, PW_POW, PW_TANH_BACKWARD,
 PW_SIGMOID_BACKWARD) = range(16, 28)
PW_IMM, PW_T0, PW_SCALAR, PW_CHANNEL, PW_ROW, PW_DM, PW_M = range(7)  # (DM, M: the general layout's g only)
PW_SRK_MAX_REGS = 18  # TSDE_PW_SRK_MAX_REGS
KERNEL_PW_MILSTEIN = 3  # TSDE_KERNEL_PW_MILSTEIN
KERNEL_PW_SRK = 4  # TSDE_KERNEL_PW_SRK
KERNEL_PW_PC = 5  # TSDE_KERNEL_PW_PC
KERNEL_PW_CHUNK = 6  # TSDE_KERNEL_PW_CHUNK
KERNEL_PW_ADAPTIVE = 7  # TSDE_KERNEL_PW_ADAPTIVE
KERNEL_PW_GENERAL = 8  # TSDE_KERNEL_PW_GENERAL
KERNEL_PW_ADJOINT = 9  # TSDE_KERNEL_PW_ADJOINT
PW_GENERAL_MAX_M = 32  # TSDE_PW_GENERAL_MAX_M
PW_LAYOUT_GENERAL = 1  # TSDE_PW_LAYOUT_GENERAL: Pointwise.reserved of a general-noise program
PW_LAYOUT_GENERAL_SRA = 2  # TSDE_PW_LAYOUT_GENERAL_SRA: Pointwise.reserved of a general-noise program of an sra1 step
PW_LAYOUT_GENERAL_EULER_HEUN = 3  # TSDE_PW_LAYOUT_GENERAL_EULER_HEUN: ... of a general-noise Euler-Heun step
PW_LAYOUT_GENERAL_REVERSIBLE_HEUN = 4  # TSDE_PW_LAYOUT_GENERAL_REVERSIBLE_HEUN: ... of general reversible-Heun chunks
# TSDE_PROPOSAL_*: the method of tsde_adaptive_proposal_pointwise
(PROPOSAL_EULER, PROPOSAL_MILSTEIN_ITO, PROPOSAL_MILSTEIN_STRATONOVICH, PROPOSAL_SRK, PROPOSAL_HEUN, PROPOSAL_MIDPOINT,
 PROPOSAL_EULER_HEUN) = range(7)
PC_HEUN, PC_MIDPOINT, PC_EULER_HEUN = range(3)  # TSDE_PC_*
PW_MAX_STEPS = 64  # TSDE_PW_MAX_STEPS
PW_ADJ_MAX_PARAMS = 8  # TSDE_PW_ADJ_MAX_PARAMS
PW_SRC_GO2 = 0xFD  # TSDE_PW_SRC_GO2: the adjoint layout's second vjp seed (g's cotangent)
PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN = 5  # TSDE_PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN: ... of a PwAdjoint's program


class PwInstr(ctypes.Structure):
    _fields_ = [('op', ctypes.c_uint8), ('dst', ctypes.c_uint8), ('a', ctypes.c_uint8), ('b', ctypes.c_uint8)]


class PwOperand(ctypes.Structure):
    _fields_ = [('kind', ctypes.c_int32), ('reserved', ctypes.c_int32), ('ptr', ctypes.c_void_p),
                ('imm', ctypes.c_double)]


class Pointwise(ctypes.Structure):
    _fields_ = [('n_instr', ctypes.c_int32), ('n_fg', ctypes.c_int32), ('n_regs', ctypes.c_int32),
                ('n_operands', ctypes.c_int32), ('f_src', ctypes.c_uint8), ('g_src', ctypes.c_uint8),
                ('gdg_src', ctypes.c_uint8), ('reserved', ctypes.c_uint8),
                ('instr', PwInstr * PW_MAX_INSTR), ('operand', PwOperand * PW_MAX_OPERANDS)]


class PwStep(ctypes.Structure):
    _fields_ = [('cell_id', ctypes.c_uint64), ('h', ctypes.c_double), ('dt', ctypes.c_double), ('t0', ctypes.c_void_p),
                ('y1', ctypes.c_void_p)]


class PwAdjoint(ctypes.Structure):
    """tsde_pw_adjoint: a program tagged PW_LAYOUT_ADJOINT_REVERSIBLE_HEUN and the buffers of one launch (the entry
    points take `prog`, the first member)."""
    _fields_ = [('prog', Pointwise), ('n_params', ctypes.c_int32), ('reserved', ctypes.c_int32),
                ('param_src', ctypes.c_uint8 * PW_ADJ_MAX_PARAMS), ('t0', ctypes.c_void_p),
                ('adj_in', ctypes.c_void_p * 4), ('y1', ctypes.c_void_p), ('adj_out', ctypes.c_void_p * 4),
                ('ys', ctypes.c_void_p), ('grad_ys', ctypes.c_void_p), ('n_out', ctypes.c_int64),
                ('partial', ctypes.c_void_p * PW_ADJ_MAX_PARAMS)]


class PwSubstep(ctypes.Structure):
    _fields_ = [('w', ctypes.c_void_p), ('u', ctypes.c_void_p), ('t', ctypes.c_void_p * 4), ('dt', ctypes.c_double),
                ('s', ctypes.c_double * 3)]


_P = ctypes.c_void_p
_D = ctypes.c_double
_I = ctypes.c_int32
_L = ctypes.POINTER(Launch)
_N = ctypes.POINTER(Noise)

# name -> argtypes after (launch, [noise]).  Mirrors include/torchsde_b200.h one to one.
SIGNATURES = {
    'tsde_brownian_cells': [_L, _N, _P, _P, _P],
    'tsde_brownian_bridge': [_L, _P, ctypes.c_int64, _I, ctypes.POINTER(ctypes.c_uint64),
                             ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_double), _P, _P, _P, _P],
    'tsde_brownian_merge': [_L, _P, _P, _P, _P, _D, _D, _D],
    'tsde_brownian_h_to_u': [_L, _P, _P, _D, _P],
    'tsde_brownian_levy_area': [_L, _P, ctypes.c_int64, ctypes.c_uint64, _P, _P, _D, _I, _P],
    'tsde_brownian_merge_area': [_L, _P, _P, _P, _P],
    'tsde_bmm_ga': [_L, _P, _P, _P],
    'tsde_logqp_augment': [_L, _P, _P, _P, _D, _P, _P],
    'tsde_brownian_cell_levy': [_L, _N, ctypes.c_uint64, _I, _P, _P, _P],
    'tsde_step_euler': [_L, _N, _P, _P, _P, _D, _P],
    'tsde_milstein_vjp_seed': [_L, _N, _P, _D, _I, _P],
    'tsde_step_milstein': [_L, _N, _P, _P, _P, _P, _D, _P],
    'tsde_step_milstein_pointwise': [_L, _N, ctypes.POINTER(Pointwise), _P, _P, _D, _I, _P],
    'tsde_solve_milstein_pointwise': [_L, _N, ctypes.POINTER(Pointwise), _P, ctypes.POINTER(PwStep), _I, _I],
    'tsde_pointwise_compile': [_L, ctypes.POINTER(Pointwise)],
    'tsde_pointwise_source': [_L, ctypes.POINTER(Pointwise), ctypes.c_char_p, ctypes.c_int64],
    'tsde_step_srk_diag_pointwise': [_L, _N, ctypes.POINTER(Pointwise), _P, _P, _P, _P, _P, _D, _D, _D, _D, _P],
    'tsde_step_predictor_corrector_pointwise': [_L, _N, ctypes.POINTER(Pointwise), _P, _P, _P, _I, _D, _D, _P],
    'tsde_solve_euler_pointwise': [_L, _N, ctypes.POINTER(Pointwise), _P, ctypes.POINTER(PwStep), _I],
    'tsde_solve_reversible_heun_pointwise': [_L, _N, ctypes.POINTER(Pointwise), _P, _P, _P, _P,
                                             ctypes.POINTER(PwStep), _I, _P, _P, _P],
    'tsde_adaptive_proposal_pointwise': [_L, ctypes.POINTER(Pointwise), _I, _P, ctypes.POINTER(PwSubstep), _P, _P],
    'tsde_adaptive_pointwise_compile': [_L, ctypes.POINTER(Pointwise)],
    'tsde_milstein_gf_predict': [_L, _P, _P, _P, _D, _D, _I, _P],
    'tsde_step_milstein_gf': [_L, _N, _P, _P, _P, _P, _D, _D, _I, _P],
    'tsde_step_heun': [_L, _N, _P, _P, _P, _P, _P, _D, _P],
    'tsde_midpoint_predict': [_L, _N, _P, _P, _P, _D, _P],
    'tsde_euler_heun_predict': [_L, _N, _P, _P, _P],
    'tsde_step_euler_heun': [_L, _N, _P, _P, _P, _P, _D, _P],
    'tsde_reversible_heun_z': [_L, _N, _P, _P, _P, _P, _D, _P],
    'tsde_step_reversible_heun': [_L, _N, _P, _P, _P, _P, _P, _D, _P],
    'tsde_srk_diag_stage1': [_L, _P, _P, _P, _D, _D, _P, _P],
    'tsde_srk_diag_stage2': [_L, _N, _P, _P, _P, _P, _P, _D, _D, _D, _P, _P],
    'tsde_srk_diag_stage3': [_L, _P, _P, _P, _P, _P, _D, _D, _P],
    'tsde_step_srk_diag': [_L, _N, _P, _P, _P, _P, _P, _P, _P, _P, _D, _D, _D, _D, _P],
    'tsde_srk_additive_stage': [_L, _N, _P, _P, _P, _D, _D, _P],
    'tsde_step_srk_additive': [_L, _N, _P, _P, _P, _P, _P, _D, _D, _P],
    'tsde_linear_interp': [_L, _P, _P, _D, _D, _P],
    'tsde_adaptive_error_sumsq': [_L, _P, _P, _D, _D, _D, _P, _P],
    'tsde_adjoint_reversible_heun_a': [_L, _N, _P, _P, _P, _P, _P, _P, _P, _D, _D, _P, _P, _P],
    'tsde_adjoint_reversible_heun_b': [_L, _N, _P, _P, _P, _P, _P, _P, _P, _P, _D, _D, _P, _P, _P, _P, _P],
}

_lib = None


def _preload(package, name):
    """Load `name` from the nvidia package `package` PyTorch installs, if there is one, so that the library's dlopen
    finds it; the handle, or None."""
    try:
        pkg = importlib.import_module(f'nvidia.{package}')
    except ImportError:
        return None
    for d in getattr(pkg, '__path__', ()):
        path = os.path.join(d, 'lib', name)
        if os.path.exists(path):
            try:
                return ctypes.CDLL(path, mode=ctypes.RTLD_GLOBAL)
            except OSError:
                continue
    return None


def _preload_nvrtc():
    """Load NVRTC from the nvidia-cuda-nvrtc package PyTorch installs, if there is one, so that the library's
    dlopen("libnvrtc.so.12") finds it when the Milstein programs are compiled (tsde_pointwise_compile).  Without it the
    library still loads, and those solves keep the unfused step."""
    _preload('cuda_nvrtc', 'libnvrtc.so.12')


_nvjitlink = None


def nvjitlink():
    """nvJitLink, which links the programs with transcendental ops, loaded (once) from the nvidia-nvjitlink package
    PyTorch installs, else from the library path, so that the library's dlopen("libnvJitLink.so.12") finds it; None
    if there is none.  Only a solve that records a transcendental op loads it."""
    global _nvjitlink
    if _nvjitlink is None:
        _nvjitlink = _preload('nvjitlink', 'libnvJitLink.so.12')
        if _nvjitlink is None:
            try:
                _nvjitlink = ctypes.CDLL('libnvJitLink.so.12', mode=ctypes.RTLD_GLOBAL)
            except OSError:
                return None
    return _nvjitlink


def nvrtc_version():
    """(major, minor) of the NVRTC the library compiles programs with (the libnvrtc.so.12 its dlopen finds: the
    package's, preloaded), or None if there is none."""
    lib()
    try:
        nv = ctypes.CDLL('libnvrtc.so.12')
    except OSError:
        return None
    major, minor = ctypes.c_int(), ctypes.c_int()
    if nv.nvrtcVersion(ctypes.byref(major), ctypes.byref(minor)) != 0:
        return None
    return major.value, minor.value


def lib():
    """Load the shared library (once) and attach prototypes."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LibraryNotBuilt(
            f"torchsde_b200: CUDA library not found at {LIB_PATH}. Build it with "
            f"`python -c 'import __graft_entry__ as g; g.build()'` from the repository root. "
            f"There is no CPU or PyTorch fallback.")
    _preload_nvrtc()
    handle = ctypes.CDLL(LIB_PATH)
    handle.tsde_abi_version.restype = ctypes.c_int
    handle.tsde_error_string.restype = ctypes.c_char_p
    handle.tsde_error_string.argtypes = [ctypes.c_int]
    handle.tsde_kernel_launches.restype = ctypes.c_int64
    handle.tsde_kernel_launches.argtypes = [ctypes.c_int32]
    for name, argtypes in SIGNATURES.items():
        fn = getattr(handle, name)  # AttributeError here = header/library mismatch: fail loudly
        fn.restype = ctypes.c_int
        fn.argtypes = argtypes
    handle.tsde_pointwise_source.restype = ctypes.c_int64
    if handle.tsde_abi_version() != 1:
        raise LibraryNotBuilt("torchsde_b200: ABI version mismatch, rebuild the library.")
    _lib = handle
    return _lib


LAUNCHES = 0  # number of C-ABI launch calls issued by this process (bench.py reports it)


def check(code, what):
    global LAUNCHES
    LAUNCHES += 1
    if code != 0:
        msg = lib().tsde_error_string(code).decode()
        raise RuntimeError(f"torchsde_b200: {what} failed: {msg} (code {code})")


def dtype_code(dtype):
    if dtype == torch.float32:
        return F32
    if dtype == torch.float64:
        return F64
    raise ValueError(f"torchsde_b200 supports float32 and float64 tensors, got {dtype}.")


FMT_STATE, FMT_BF16, FMT_F16 = 0, 1, 2
_FMT = {torch.bfloat16: FMT_BF16, torch.float16: FMT_F16}

# entry point -> its tensor inputs, in declaration order.  Those named in SDE_OUTPUT_NAMES hold what the user's drift /
# diffusion returned and may be 16-bit (torch.autocast); every other input has the state dtype.
INPUTS = {
    'tsde_step_euler': ('y0', 'f', 'g'),
    'tsde_milstein_vjp_seed': ('g',),
    'tsde_step_milstein': ('y0', 'f', 'g', 'gdg'),
    'tsde_adaptive_proposal_pointwise': [_L, ctypes.POINTER(Pointwise), _I, _P, ctypes.POINTER(PwSubstep), _P, _P],
    'tsde_adaptive_pointwise_compile': [_L, ctypes.POINTER(Pointwise)],
    'tsde_milstein_gf_predict': ('y0', 'f', 'g'),
    'tsde_step_milstein_gf': ('y0', 'f', 'g', 'gp'),
    'tsde_step_heun': ('y0', 'f', 'fp', 'g', 'gp'),
    'tsde_midpoint_predict': ('y0', 'f', 'g'),
    'tsde_euler_heun_predict': ('y0', 'g'),
    'tsde_step_euler_heun': ('y0', 'f', 'g', 'gp'),
    'tsde_reversible_heun_z': ('y0', 'z0', 'f0', 'g0'),
    'tsde_step_reversible_heun': ('y0', 'f0', 'f1', 'g0', 'g1'),
    'tsde_srk_diag_stage1': ('y0', 'f0', 'g0'),
    'tsde_srk_diag_stage2': ('y0', 'f0', 'g0', 'f1', 'g1'),
    'tsde_srk_diag_stage3': ('y0', 'g0', 'g1', 'f2', 'g2'),
    'tsde_step_srk_diag': ('y0', 'f0', 'f1', 'f2', 'g0', 'g1', 'g2', 'g3'),
    'tsde_srk_additive_stage': ('y0', 'f0', 'ga'),
    'tsde_step_srk_additive': ('y0', 'f0', 'f1', 'ga', 'gb'),
    'tsde_adjoint_reversible_heun_a': ('y0', 'z0', 'f0', 'g0', 'adj_y0', 'adj_f0', 'adj_g0'),
    'tsde_adjoint_reversible_heun_b': ('y0', 'f0', 'f1', 'g0', 'g1', 'adj_y0', 'adj_z0', 'vjp_z'),
    'tsde_linear_interp': ('y0', 'y1'),
}
SDE_OUTPUT_NAMES = frozenset(('f', 'f0', 'f1', 'f2', 'fp', 'g', 'g0', 'g1', 'g2', 'g3', 'gp', 'ga', 'gb'))


def operands(name, state_dtype, ins):
    """(tsde_launch.dtype, inputs) of a launch of `name` whose state has `state_dtype`.  A bf16 / fp16 SDE output is
    passed as it is with its format bits (float32 state) or widened exactly to float64 (float64 state); any other
    dtype mismatch is a ValueError."""
    word = dtype_code(state_dtype)
    if all(t.dtype == state_dtype for t in ins):
        return word, ins
    out = list(ins)
    for i, (arg, t) in enumerate(zip(INPUTS[name], ins)):
        if t.dtype == state_dtype:
            continue
        fmt = _FMT.get(t.dtype) if arg in SDE_OUTPUT_NAMES else None
        if fmt is None:
            what = 'the SDE returned' if arg in SDE_OUTPUT_NAMES else 'got'
            raise ValueError(f"torchsde_b200: `{arg}` of {name} has dtype {t.dtype}, but the state is {state_dtype}; "
                             f"{what} a tensor that is neither the state dtype nor bfloat16 / float16.")
        if state_dtype == torch.float64:
            out[i] = t.to(torch.float64)
        else:
            word |= fmt << (8 + 2 * i)
    return word, out


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                "torchsde_b200 is a CUDA (sm_90a) implementation: tensors must live on a CUDA device. "
                "There is no CPU path; use the reference torchsde for CPU solves.")


def make_launch(dtype, noise_type, rows, d, m, stream=None, device=None):
    if stream is None:
        stream = torch.cuda.current_stream(device).cuda_stream  # the stream of the tensors' device, not of the current one
    return Launch(dtype_code(dtype), noise_type, rows, d, m, stream)


def device_guard(device):
    """Make `device` the current CUDA device for the duration of a solve / query: the C ABI launches on the stream
    it is handed and never calls cudaSetDevice, and a launch on a stream of another device than the current one
    is an invalid resource handle.  No-op for non-CUDA devices (the host-side dry runs of the test-suite)."""
    import contextlib
    device = torch.device(device) if device is not None else None
    if device is None or device.type != 'cuda':
        return contextlib.nullcontext()
    return torch.cuda.device(device)


class nvtx_range:
    """NVTX range around a host-side phase (solve, graph capture, replay, backward sweep) when TSDE_NVTX=1 — what
    shows up as named spans on an Nsight Systems timeline (SURVEY §5: tracing).  Free when the variable is unset."""
    _on = os.environ.get('TSDE_NVTX', '0') not in ('0', '')

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if self._on:
            torch.cuda.nvtx.range_push(self.name)

    def __exit__(self, *exc):
        if self._on:
            torch.cuda.nvtx.range_pop()


def ptr(t):
    """Device pointer of a contiguous tensor (or NULL)."""
    if t is None:
        return None
    if not t.is_contiguous():
        raise RuntimeError("torchsde_b200: internal error, non-contiguous tensor at the C ABI.")
    return t.data_ptr()
