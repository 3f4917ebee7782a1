"""Static SASS evidence for the shipped library (no GPU needed): per kernel family, registers / spills and the
counts of the instructions that carry the design — 128-bit global loads/stores, evict-first loads, bulk copies
(UBLKCP) and mbarrier ops (SYNCS) of the TMA-staged tile kernel, SFU ops of the in-register Box-Muller, and the
absence of FFMA in the tableau kernels that follow the reference's separately rounded op order (-fmad=false).  In the
chunked Euler / reversible-Heun kernels it checks the element-wise program's interpreter loops (the innermost loops that
load and store the shared-memory register file): the loop that runs programs whose operands all sit in shared memory
reads no global memory (LDG) and decodes no byte fields from the parameter space (LDC.U8).  Milstein programs are not
interpreted but compiled at run time (NVRTC): it writes cfg2's program out (tsde_pointwise_source), compiles it as the
library does and checks that the compiled kernel's step loop touches no shared memory (LDS / STS), no local memory
(LDL / STL, spills) and reads no instruction word from the parameter space (an indexed LDC).  Its loops for a uniform
grid (PwSteps::uniform, one per `ito`) each have one back-edge, no indexed LDC / ULDC, no LDL / STL and at most
UNIFORM_MAX instructions, and the kernel at most 64 registers (its launch bounds, 256 threads x 4 CTAs); exit status 1
otherwise.

    python profiles/sass_check.py > out/sass_evidence.txt
"""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'torchsde_b200', 'lib', 'libtorchsde_b200.so')
PICK = [  # (label, regex on the demangled kernel name)
    ('Milstein tableau, fp32, counter noise (headline)', r'ew_fast_kernel<float, tsde::MilsteinOp<float>, 1>'),
    ('fused SRK step of an element-wise SDE (interpreter), fp32, counter noise', r'pw_srk_kernel<float, 1>'),
    ('fused SRK step of an element-wise SDE (interpreter), fp64, counter noise', r'pw_srk_kernel<double, 1>'),
    ('fused Heun step of an element-wise SDE (interpreter), fp32, counter noise', r'pw_pc_kernel<float, 1, 0>'),
    ('fused midpoint step of an element-wise SDE (interpreter), fp64, counter noise', r'pw_pc_kernel<double, 1, 1>'),
    ('fused Euler steps of an element-wise SDE, up to 64 per launch (interpreter), fp32, counter noise',
     r'pw_chunk_kernel<float, 1, 0>'),
    ('fused reversible-Heun steps of an element-wise SDE, up to 64 per launch (interpreter), fp32, counter noise',
     r'pw_chunk_kernel<float, 1, 1>'),
    ('fused reversible-Heun steps of an element-wise SDE, up to 64 per launch (interpreter), fp64, counter noise',
     r'pw_chunk_kernel<double, 1, 1>'),
    ('Milstein vjp seed, fp32, counter noise', r'ew_fast_kernel<float, tsde::MilsteinVjpSeedOp<float>, 1>|ew_fast_kernel<float, tsde::MilsteinSeedOp<float>, 1>'),
    ('SRK srid2 final stage, fp32', r'ew_fast_kernel<float, tsde::SrkDiagFinalOp<float>, 1>'),
    ('Euler tableau, fp64, counter noise', r'ew_fast_kernel<double, tsde::EulerOp<double>, 1>'),
    ('general Euler tile, per-thread loads, fp32', r'gen_cta_kernel<float, tsde::GEulerOp<float>, 1>'),
    ('general Heun tile, per-thread loads, fp32', r'gen_cta_kernel<float, tsde::GHeunOp<float>, 1>'),
    ('general Euler tile, TMA-staged, fp32, m=16', r'gen_tma_kernel<float, tsde::GEulerOp<float>, 1, 2>'),
    ('general Heun tile, TMA-staged, fp32, m=64', r'gen_tma_kernel<float, tsde::GHeunOp<float>, 1, 4>'),
    ('general Euler tile, wide rows (m in chunks), fp32', r'gen_wide_kernel<float, tsde::GEulerOp<float>, 1>'),
    ('general SRK-additive final tile, wide rows, fp64', r'gen_wide_kernel<double, tsde::GSraFinalOp<double>, 1>'),
    ('Brownian cells W (materialised queries), fp32', r'ew_fast_kernel<float, tsde::CellsOp<float, false>, 1>|ew_fast_kernel<float, tsde::CellsOp<float>, 1>'),
    ('Brownian bridge', r'bridge_kernel<float'),
    ('Levy area (Davie / Foster), fp32, m = 16: one normal per pair, pair arithmetic two at a time', r'levy_tile_kernel<float, false, 16>|levy_tile_kernel<float, \(bool\)0, 16>'),
    ('fused cell query W, U, A (drawn in the kernel), fp32, m = 16', r'levy_tile_kernel<float, true, 16>|levy_tile_kernel<float, \(bool\)1, 16>'),
    ('Levy area, fp64, m = 16 (scalar pair arithmetic, separately rounded)', r'levy_tile_kernel<double, false, 16>|levy_tile_kernel<double, \(bool\)0, 16>'),
    ('bmm(g, A) of the log-ODE correction, fp32, m = 16', r'bmm_ga_kernel<float, 16>'),
    ('logqp KL-integrand augmentation, fp32', r'logqp_augment_kernel<float>'),
]
INTERPRETED = [r'pw_chunk_kernel<float, 1, 0>', r'pw_chunk_kernel<double, 1, 0>', r'pw_chunk_kernel<float, 1, 1>', r'pw_chunk_kernel<double, 1, 1>']
UNIFORM_MAX = 150  # instructions per step of the uniform-grid loop (one back-edge: the static count is the dynamic one)
COUNT = ['LDG.E.128', 'LDG.E.EF.128', 'STG.E.128', 'LDS.128', 'UBLKCP', 'SYNCS', 'MUFU', 'FFMA', 'FMUL', 'FADD', 'DFMA',
         'SHFL', 'BAR.SYNC', 'LDL', 'STL', 'IMAD.WIDE']


def interpreter_loops(sass):
    """The innermost loops (a backward branch and its target, holding no other backward branch) that load and store
    the shared-memory register file, as lists of instructions."""
    ins = []
    for ln in sass.splitlines():
        m = re.match(r'\s+/\*([0-9a-f]{4,})\*/\s+(.*?);', ln)
        if m:
            ins.append((int(m.group(1), 16), m.group(2)))
    back = []
    for i, (addr, op) in enumerate(ins):
        m = re.search(r'\bBRA\s+(?:`\()?0x([0-9a-f]+)', op)
        if m and int(m.group(1), 16) < addr:
            back.append((int(m.group(1), 16), addr))
    inner = [(a, b) for a, b in back if not any(a <= c < d <= b and (c, d) != (a, b) for c, d in back)]
    loops = [[op for addr, op in ins if a <= addr <= b] for a, b in inner]
    return [body for body in loops if any('LDS.128' in o for o in body) and any('STS.128' in o for o in body)]


def compiled_milstein():
    """cfg2's Milstein program as the library compiles it: its step loop, registers and spills; False if it fails."""
    import tempfile
    sys.path.insert(0, ROOT)
    import torch
    from tests import test_host_pointwise as milstein
    from tests.test_host_pointwise_compile import OPTIONS, HEADERS, STDINT, _tape
    from torchsde_b200 import _cabi
    import ctypes
    src = _cabi.pointwise_source(_tape(milstein.ACCEPTED, 'gbm_ito', torch.float32), torch.float32)
    nv = ctypes.CDLL('libnvrtc.so.12')
    arr = lambda xs: (ctypes.c_char_p * len(xs))(*[x.encode() for x in xs])  # noqa: E731
    prog = ctypes.c_void_p()
    names = list(HEADERS) + ['stdint.h']
    nv.nvrtcCreateProgram(ctypes.byref(prog), src.encode(), b'cfg2.cu', len(names),
                          arr([open(p).read() for p in HEADERS.values()] + [STDINT]), arr(names))
    assert nv.nvrtcCompileProgram(prog, len(OPTIONS), arr(OPTIONS)) == 0
    n = ctypes.c_size_t()
    nv.nvrtcGetCUBINSize(prog, ctypes.byref(n))
    cubin = ctypes.create_string_buffer(n.value)
    nv.nvrtcGetCUBIN(prog, cubin)
    with tempfile.NamedTemporaryFile(suffix='.cubin') as f:
        f.write(cubin.raw)
        f.flush()
        res = subprocess.run(['cuobjdump', '-res-usage', f.name], capture_output=True, text=True).stdout
        sass = subprocess.run(['cuobjdump', '-sass', '-fun', 'tsde_pw_milstein_single', f.name], capture_output=True,
                              text=True).stdout
    m = re.search(r'Function tsde_pw_milstein_single:\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)', res)
    reg, stack, shared, local = (int(m.group(i)) for i in range(1, 5))
    ins = []
    for ln in sass.splitlines():
        mm = re.match(r'\s+/\*([0-9a-f]{4,})\*/\s+(.*?);', ln)
        if mm:
            ins.append((int(mm.group(1), 16), mm.group(2)))
    back = [(int(re.search(r'0x([0-9a-f]+)', op.split('BRA')[1]).group(1), 16), addr) for addr, op in ins
            if re.search(r'\bBRA\b', op) and re.search(r'0x([0-9a-f]+)', op.split('BRA')[1])
            and int(re.search(r'0x([0-9a-f]+)', op.split('BRA')[1]).group(1), 16) < addr]
    a, b = max(back, key=lambda x: x[1] - x[0])  # the step table's loop: the outermost backward branch
    loop = [op for addr, op in ins if a <= addr <= b]
    bad = [o for o in loop if re.search(r'\bLDS|\bSTS|\bLDL|\bSTL|LDC[.\w]*\s+\S+,\s*c\[0x0\]\[R', o)]
    cnt = {k: sum(1 for o in loop if re.search(r'\b' + re.escape(k) + r'\b', o)) for k in COUNT}
    print(f"## cfg2's Milstein program, compiled at run time (NVRTC), fp32, one cell per step\n"
          f"   REG {reg}  STACK {stack}  SHARED {shared}  LOCAL {local}  step-table loop: {len(loop)} instructions\n   " +
          '  '.join(f"{k}={v}" for k, v in cnt.items() if v) +
          f"\n   shared / local memory or indexed parameter reads in the step-table loop: {len(bad)}")
    # the uniform-grid loops: the loops whose only branch is their back-edge
    uniform = [[op for addr, op in ins if x <= addr <= y] for x, y in back]
    uniform = [u for u in uniform if sum(1 for o in u if re.search(r'\bBRA\b', o)) == 1]
    ok = len(uniform) == 2 and reg <= 64
    for u in uniform:
        ubad = [o for o in u if re.search(r'\bLDL|\bSTL|U?LDC[.\w]*\s+\S+,\s*c\[0x0\]\[U?R', o)]
        ok = ok and not ubad and len(u) <= UNIFORM_MAX
        cnt = {k: sum(1 for o in u if re.search(r'\b' + re.escape(k) + r'\b', o)) for k in COUNT}
        print(f"   uniform-grid loop: {len(u)} instructions (at most {UNIFORM_MAX}), indexed parameter reads or local"
              f" memory: {len(ubad)}\n   " + '  '.join(f"{k}={v}" for k, v in cnt.items() if v))
    print(f"   uniform-grid loops: {len(uniform)} (one per ito), registers {reg} (at most 64)\n")
    return ok and not bad and not stack and not local


# The general-noise adjoint kernel (pw_general_adjoint_reversible_heun_steps) of correlated GBM (f = mu*y,
# g = y.unsqueeze(-1) * S): (m, dtype) -> the most spill memory (bytes per thread, STACK + LOCAL of cuobjdump
# -res-usage) its single- and multi-cell kernels may use, as measured with CUDA 12.9.  It keeps no (d, m) block in registers, but the four lanes' channel passes,
# the step's increments w and the previous step's wp stay live together; past m = 8 in fp32 and m = 4 in fp64 the
# 255 registers of its launch bounds (256, 1) do not hold them (DESIGN section 3).
GENERAL_ADJOINT_SPILL = {(4, 'float32'): 0, (16, 'float32'): 8, (32, 'float32'): 8,
                         (4, 'float64'): 0, (16, 'float64'): 64, (32, 'float64'): 832}


def _nvrtc_usage(src, kernels):
    """{kernel: (REG, STACK, LOCAL)} of `src` compiled as the library compiles a program (NVRTC, its options)."""
    import ctypes
    import tempfile
    from tests.test_host_pointwise_compile import OPTIONS, HEADERS, STDINT
    nv = ctypes.CDLL('libnvrtc.so.12')
    arr = lambda xs: (ctypes.c_char_p * len(xs))(*[x.encode() for x in xs])  # noqa: E731
    prog = ctypes.c_void_p()
    names = list(HEADERS) + ['stdint.h']
    nv.nvrtcCreateProgram(ctypes.byref(prog), src.encode(), b'prog.cu', len(names),
                          arr([open(p).read() for p in HEADERS.values()] + [STDINT]), arr(names))
    assert nv.nvrtcCompileProgram(prog, len(OPTIONS), arr(OPTIONS)) == 0
    n = ctypes.c_size_t()
    nv.nvrtcGetCUBINSize(prog, ctypes.byref(n))
    cubin = ctypes.create_string_buffer(n.value)
    nv.nvrtcGetCUBIN(prog, cubin)
    with tempfile.NamedTemporaryFile(suffix='.cubin') as f:
        f.write(cubin.raw)
        f.flush()
        res = subprocess.run(['cuobjdump', '-res-usage', f.name], capture_output=True, text=True).stdout
    out = {}
    for k in kernels:
        m = re.search(r'Function ' + k + r':\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)', res)
        out[k] = (int(m.group(1)), int(m.group(2)), int(m.group(4)))
    return out


def compiled_general_adjoint():
    """Registers and local memory of the general-noise adjoint kernels at m = 4, 16, 32 in fp32 and fp64, against
    GENERAL_ADJOINT_SPILL; False if one spills more than it states."""
    sys.path.insert(0, ROOT)
    import torch
    from tests import test_host_pointwise_adjoint_general as gen
    from torchsde_b200 import _cabi
    ok = True
    print("## the general-noise adjoint's backward-step kernel (correlated GBM), compiled at run time (NVRTC)\n"
          "   m  dtype     single: REG STACK LOCAL   multi: REG STACK LOCAL   (STACK + LOCAL at most)")
    for dtype in (torch.float32, torch.float64):
        for m in (4, 16, 32):
            mu = gen.P(gen.D).detach().to(dtype).requires_grad_()
            S = gen.P(gen.D, m).detach().to(dtype).requires_grad_()
            rec, res = gen.record(lambda t, y: mu * y, lambda t, y: y.unsqueeze(-1) * S, [mu, S], m=m, dtype=dtype)
            src = _cabi.general_pointwise_source(res[0].prog, dtype, gen.D, m)
            names = ['tsde_pw_general_adjoint_reversible_heun_single', 'tsde_pw_general_adjoint_reversible_heun_multi']
            u = _nvrtc_usage(src, names)
            name = str(dtype).split('.')[-1]
            most = GENERAL_ADJOINT_SPILL[(m, name)]
            ok = ok and all(v[1] + v[2] <= most for v in u.values())
            print(f"   {m:2d} {name}   {u[names[0]][0]:3d} {u[names[0]][1]:5d} {u[names[0]][2]:5d}           "
                  f"{u[names[1]][0]:3d} {u[names[1]][1]:5d} {u[names[1]][2]:5d}   ({most})")
    print()
    return ok


def main():
    if not os.path.exists(LIB):
        sys.exit("build the library first: python -c 'import __graft_entry__ as g; g.build()'")
    res = subprocess.run(['cuobjdump', '-res-usage', LIB], capture_output=True, text=True).stdout
    usage = {}
    for m in re.finditer(r'Function (\S+):\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)', res):
        usage[m.group(1)] = tuple(int(m.group(i)) for i in range(2, 6))
    names = sorted(usage)
    dem = subprocess.run(['c++filt'], input='\n'.join(names), capture_output=True, text=True).stdout.splitlines()
    framed = [(n, d) for n, d in zip(names, dem) if usage[n][1] or usage[n][3]]
    f32 = [d for n, d in framed if '<float' in d]
    print(f"library: {os.path.relpath(LIB, ROOT)}   kernels: {len(names)}   max registers: {max(u[0] for u in usage.values())}")
    print(f"kernels with a stack frame: {len(framed)} (fp64 libm slow paths of log / sincospi), of which fp32: {len(f32)}")
    fam = {}
    for d in f32:
        k = d.split('(')[0].split('<')[0].replace('void ', '')
        fam[k] = fam.get(k, 0) + 1
    for k, v in sorted(fam.items()):
        print(f"   fp32 with a stack frame: {k} x{v}")
    print("   (small frames: generic fallback kernels, and the increment staging of gen_tma_kernel's producer warp — none on a"
          " hot loop; the specialised ew_fast_kernel / gen_cta_kernel instantiations have none)")
    print()
    for label, pat in PICK:
        hit = [(n, d) for n, d in zip(names, dem) if re.search(pat, d)]
        if not hit:
            print(f"## {label}\n   (no kernel matches /{pat}/)\n")
            continue
        n, d = hit[0]
        sass = subprocess.run(['cuobjdump', '-sass', '-fun', n, LIB], capture_output=True, text=True).stdout
        ops = [ln.split(';')[0] for ln in sass.splitlines() if re.match(r'\s+/\*[0-9a-f]{4,}\*/', ln)]
        reg, stack, shared, local = usage[n]
        print(f"## {label}\n   {d.split('(')[0]}\n   instructions {len(ops)}  REG {reg}  STACK {stack}  SHARED(static) {shared}  LOCAL {local}")
        cnt = {k: sum(1 for o in ops if re.search(r'\b' + re.escape(k) + r'\b', o)) for k in COUNT}
        print('   ' + '  '.join(f"{k}={v}" for k, v in cnt.items() if v) + '\n')
    bad = 0 if compiled_milstein() else 1
    bad += 0 if compiled_general_adjoint() else 1
    for pat in INTERPRETED:
        hit = [n for n, d in zip(names, dem) if re.search(pat, d)]
        sass = subprocess.run(['cuobjdump', '-sass', '-fun', hit[0], LIB], capture_output=True, text=True).stdout
        loops = interpreter_loops(sass)
        clean = [b for b in loops if not any(re.search(r'\bLDG\b|\bLDC\.U8\b', o) for o in b)]
        sizes = ', '.join(str(len(b)) for b in clean)
        print(f"## interpreter loops of {pat}: {len(loops)}, of which {len(clean)} read only shared memory and the"
              f" instruction word ({sizes} instructions)")
        bad += not clean
    sys.exit(1 if bad else 0)


if __name__ == '__main__':
    main()
