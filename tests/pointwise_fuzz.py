"""A seeded generator of element-wise SDEs for the fused step programs (torchsde_b200/_core/pointwise.py).

`case(seed, layout)` draws one SDE: a random straight-line program (an expression DAG written as statements) for f and
one for g, over the state y, the time t, Python numbers and device parameters of every operand kind the recorders
know.  A `Case` is plain data: its repr is a `Case(...)` call that rebuilds it, so a failing seed can be pasted into a
regression test as it stands, and `Case.source()` prints f and g as the torch code they run.  From a case come

  * `FuzzSDE`, the nn.Module whose f and g run the statements with torch ops (`run_torch`);
  * `run_numpy`, the same statements in numpy, each op restated as ATen's CUDA kernel computes it: a division by a
    Python number is a multiplication by its reciprocal rounded to the state dtype, `x ** 2` is `x * x`, rsub swaps
    its operands, clamp is maximum then minimum, maximum / minimum propagate NaN, sign is (0 < x) - (x < 0),
    comparisons give 0 / 1 and where / masked_fill select.  The transcendental ops have no exact numpy restatement:
    a case that holds one is not `exact`.

Layouts (`LAYOUTS`): the diagonal-noise Milstein tape (f, g and autograd's vjp of g in one compiled program), the
interpreted two-program tapes of SRK ('fgfgfgg'), Heun / midpoint ('fgfg'), Euler-Heun ('fgg') and Euler / reversible
Heun ('fg'), and the general-noise tapes of Euler ('fg'), midpoint ('fgfg') and additive-noise SRK ('fggf'), whose g is
(rows, d, m).  The compiled layouts (Milstein, general) also draw the transcendental ops.

Size classes (`SIZES`): 'small' (2-6 ops per callable), 'medium' (about 20), 'limits' (wide DAGs with 14-25 values
live at once and up to 26 device operands: near TSDE_PW_MAX_INSTR, _MAX_REGS, _SRK_MAX_REGS and _MAX_OPERANDS, so some
are rejected as too long or too wide, and some operands are read from global memory past the hoisted slots) and 'edge'
(a small or medium DAG whose y0 holds 0, -0, negative values, values on and next to every comparison threshold, inf
and NaN: both sides are compared on the bits).

Every value stays in its op's domain and bounded by construction: square roots, logarithms, rsqrt and divisors read
|x| + 1/2, exp and expm1 read x clamped to [-3, 3], and a value whose bound (interval arithmetic from |y| <= 4 and
|parameter| <= 1.5) passes 8 is clamped to [-8, 8].  A 10-20-step solve from a finite y0 then stays finite.

Reproducing a seed: `print(repr(case(seed, layout)))` and `print(case(seed, layout).source())`."""
import dataclasses
import math

import numpy as np
import torch
from torch import nn

# layout -> (recorder, evaluation pattern, compiled)
LAYOUTS = {
    'milstein': ('milstein', 'fg', True),
    'srk': ('srk', 'fgfgfgg', False),
    'pc': ('srk', 'fgfg', False),
    'euler_heun': ('srk', 'fgg', False),
    'euler': ('srk', 'fg', False),
    'general_euler': ('general', 'fg', True),
    'general_midpoint': ('general', 'fgfg', True),
    'sra': ('general', 'fggf', True),
}
SIZES = ('small', 'medium', 'limits', 'edge')
ROWS, D, M = 5, 8, 5  # the host shapes; the GPU cases set their own

BMAX = 8.0   # the bound past which a value is clamped
YMAX = 4.0   # the bound assumed of y
NUMBERS = (0.5, 2.0, 3.0, 0.1, 0.7, 1.5, -0.25, 0.3, -1.0, 0.0)
DIVISORS = (3.0, 7.0, 0.1, 1.5, 10.0, 0.3, 6.0)
THRESHOLDS = (0.0, 0.5, -0.5, 0.25, 1.0)
POWERS = (0.5, -0.5, -1.0, 2.0, 3.0, -2.0, 1.5, 2.5, -1.7, 0.75)
TRANSCENDENTAL = ('exp', 'log', 'sin', 'cos', 'tanh', 'log1p', 'expm1', 'rsqrt', 'sigmoid', 'pow')

# the parameters: name prefix -> shape, as a function of (rows, d, m)
PARAM_SHAPES = {'s': lambda r, d, m: (1,), 'k': lambda r, d, m: (), 'c': lambda r, d, m: (d,),
                'r': lambda r, d, m: (r, d), 'o': lambda r, d, m: (r, d), 'q': lambda r, d, m: (d, 1),
                'w': lambda r, d, m: (m,), 'S': lambda r, d, m: (d, m)}


@dataclasses.dataclass
class Case:
    """One fuzzed SDE.  `f` and `g` are statements (target, op, args), args being names ('y', 't', a parameter, an
    earlier target) or Python numbers; `f_out` / `g_out` name the results.  Parameters: 's*' one-element device
    tensors, 'k*' 0-d tensors (CPU tensors where the state is on a GPU), 'c*' (d,), 'r*' (rows, d), 'o*' (rows, d) at
    a storage offset of one element, and for general noise 'q*' (d, 1), 'w*' (m,), 'S*' (d, m)."""
    seed: int
    layout: str
    size: str
    f: tuple
    f_out: str
    g: tuple
    g_out: str
    params: tuple
    transcendental: bool = False

    @property
    def general(self):
        return LAYOUTS[self.layout][0] == 'general'

    @property
    def exact(self):
        """Whether numpy restates every op of the case exactly (no transcendental op)."""
        return not any(op in TRANSCENDENTAL for _, op, _ in self.f + self.g)

    def source(self):
        """f and g as the torch code `run_torch` runs."""
        out = []
        for name, stmts, res in (('f', self.f, self.f_out), ('g', self.g, self.g_out)):
            out.append(f'def {name}(t, y, p):')
            out += [f'    {tgt} = {_render(op, args)}' for tgt, op, args in stmts]
            out.append(f'    return {_atom_src(res)}')
        return '\n'.join(out)


def _atom_src(a):
    if isinstance(a, str):
        return a if a in ('y', 't') or a[0] in 'vu' else f'p.{a}'
    return repr(float(a))


FORMAT = {
    'mul': '{0} * {1}', 'add': '{0} + {1}', 'sub': '{0} - {1}', 'rsub': 'torch.rsub({0}, {1})',
    'nsub': '{1} - {0}', 'div': '{0} / {1}', 'divn': '{0} / {1}', 'neg': '-{0}', 'sqrt': 'torch.sqrt({0})',
    'sq': '{0} ** 2', 'imul': '{0}.mul_({1})', 'iadd': '{0}.add_({1})',
    'lt': '{0} < {1}', 'le': '{0} <= {1}', 'gt': '{0} > {1}', 'ge': '{0} >= {1}', 'eq': '{0} == {1}',
    'ne': '{0} != {1}',
    'and': '{0} & {1}', 'or': '{0} | {1}', 'not': '~{0}',
    'where': 'torch.where({0}, {1}, {2})', 'mfill': '{0}.masked_fill({1}, {2})', 'clamp': '{0}.clamp({1}, {2})',
    'clampmin': 'torch.clamp_min({0}, {1})', 'clampmax': 'torch.clamp_max({0}, {1})',
    'clampt': 'torch.clamp({0}, min={1}, max={2})', 'clampmint': 'torch.clamp({0}, min={1})',
    'relu': 'torch.relu({0})', 'abs': '{0}.abs()', 'maximum': 'torch.maximum({0}, {1})',
    'minimum': 'torch.minimum({0}, {1})', 'recip': 'torch.reciprocal({0})', 'sign': 'torch.sign({0})',
    'exp': 'torch.exp({0})', 'log': 'torch.log({0})', 'sin': 'torch.sin({0})', 'cos': 'torch.cos({0})',
    'tanh': 'torch.tanh({0})', 'log1p': 'torch.log1p({0})', 'expm1': 'torch.expm1({0})', 'rsqrt': 'torch.rsqrt({0})',
    'sigmoid': 'torch.sigmoid({0})', 'pow': '{0} ** {1}', 'lift': '{0}.unsqueeze(-1)',
    'expand': '{0}.expand(y.size(0), y.size(1), m)',
}


def _render(op, args):
    return FORMAT[op].format(*[_atom_src(a) if isinstance(a, str) else repr(float(a)) for a in args])


# -- the two evaluators ------------------------------------------------------------------------------------------------
TORCH = {
    'mul': lambda a, b: a * b, 'add': lambda a, b: a + b, 'sub': lambda a, b: a - b, 'rsub': torch.rsub,
    'nsub': lambda a, b: b - a, 'div': lambda a, b: a / b, 'divn': lambda a, b: a / b, 'neg': lambda a: -a,
    'sqrt': torch.sqrt, 'sq': lambda a: a ** 2, 'imul': lambda a, b: a.mul_(b), 'iadd': lambda a, b: a.add_(b),
    'lt': lambda a, b: a < b, 'le': lambda a, b: a <= b, 'gt': lambda a, b: a > b, 'ge': lambda a, b: a >= b,
    'eq': lambda a, b: a == b, 'ne': lambda a, b: a != b, 'and': lambda a, b: a & b, 'or': lambda a, b: a | b,
    'not': lambda a: ~a, 'where': torch.where, 'mfill': lambda a, c, v: a.masked_fill(c, v),
    'clamp': lambda a, lo, hi: a.clamp(lo, hi), 'clampmin': torch.clamp_min, 'clampmax': torch.clamp_max,
    'clampt': lambda a, lo, hi: torch.clamp(a, min=lo, max=hi), 'clampmint': lambda a, lo: torch.clamp(a, min=lo),
    'relu': torch.relu, 'abs': lambda a: a.abs(), 'maximum': torch.maximum, 'minimum': torch.minimum,
    'recip': torch.reciprocal, 'sign': torch.sign, 'exp': torch.exp, 'log': torch.log, 'sin': torch.sin,
    'cos': torch.cos, 'tanh': torch.tanh, 'log1p': torch.log1p, 'expm1': torch.expm1, 'rsqrt': torch.rsqrt,
    'sigmoid': torch.sigmoid, 'pow': lambda a, e: a ** e, 'lift': lambda a: a.unsqueeze(-1),
}


def _nan_first(a, b, pick):
    return np.where(np.isnan(a), a, np.where(np.isnan(b), b, pick(a, b)))


def np_maximum(a, b):
    return _nan_first(a, b, np.maximum)


def np_minimum(a, b):
    return _nan_first(a, b, np.minimum)


def _numpy_ops(npt):
    one = npt(1)
    return {
        'mul': lambda a, b: a * b, 'add': lambda a, b: a + b, 'sub': lambda a, b: a - b, 'rsub': lambda a, b: b - a,
        'nsub': lambda a, b: b - a, 'div': lambda a, b: a / b, 'divn': lambda a, b: a * (one / b),
        'neg': lambda a: -a, 'sqrt': np.sqrt, 'sq': lambda a: a * a, 'imul': lambda a, b: a * b,
        'iadd': lambda a, b: a + b, 'lt': lambda a, b: a < b, 'le': lambda a, b: a <= b, 'gt': lambda a, b: a > b,
        'ge': lambda a, b: a >= b, 'eq': lambda a, b: a == b, 'ne': lambda a, b: a != b,
        'and': lambda a, b: a & b, 'or': lambda a, b: a | b, 'not': lambda a: ~a,
        'where': lambda c, a, b: np.where(c, a, b), 'mfill': lambda a, c, v: np.where(c, v, a),
        'clamp': lambda a, lo, hi: np_minimum(np_maximum(a, lo), hi), 'clampmin': np_maximum,
        'clampmax': np_minimum, 'clampt': lambda a, lo, hi: np_minimum(np_maximum(a, lo), hi),
        'clampmint': np_maximum, 'relu': lambda a: np_maximum(a, npt(0)), 'abs': np.abs,
        'maximum': np_maximum, 'minimum': np_minimum, 'recip': lambda a: one / a,
        'sign': lambda a: (npt(0) < a).astype(npt) - (a < npt(0)).astype(npt),
        'lift': lambda a: a[..., None],
    }


def run_torch(stmts, out, t, y, p, m=M):
    """The statements with torch ops (`p` holds the parameters by name; g is (rows, d, m) for general noise)."""
    env = {'y': y, 't': t}

    def get(a):
        if not isinstance(a, str):
            return a
        return env[a] if a in env else p[a]
    for tgt, op, args in stmts:
        if op == 'expand':
            env[tgt] = get(args[0]).expand(y.size(0), y.size(1), m)
            continue
        r = TORCH[op](*[get(a) for a in args])
        env[tgt] = r
        if op in ('imul', 'iadd'):
            env[args[0]] = r
    return get(out)


def run_numpy(stmts, out, t, y, p, npt, m=M):
    """The statements restated in numpy as ATen's CUDA kernels compute them; `p` holds numpy parameters.  An in-place
    op writes the storage its target shares with every earlier name of it (`v2 = v1.mul_(...)`: v1 and v2 are one
    tensor)."""
    ops = _numpy_ops(npt)
    env = {'y': y, 't': np.asarray(t, dtype=npt)}
    alias = {}  # name -> the first name of its tensor

    def get(a):
        if not isinstance(a, str):
            return npt(a)
        a = alias.get(a, a)
        return env[a] if a in env else p[a]
    with np.errstate(all='ignore'):
        for tgt, op, args in stmts:
            if op == 'expand':
                env[tgt] = np.broadcast_to(get(args[0]), y.shape + (m,))
                continue
            r = ops[op](*[get(a) for a in args])
            r = np.asarray(r) if r.dtype == np.bool_ else np.asarray(r, dtype=npt)
            if op in ('imul', 'iadd'):
                alias[tgt] = alias.get(args[0], args[0])
                env[alias[tgt]] = r
            else:
                env[tgt] = r
    return get(out)


# -- parameters ----------------------------------------------------------------------------------------------------
def param_values(case, rows, d, m, seed_shift=0):
    """float64 values of every parameter (numpy), a function of the case's seed and shapes."""
    rng = np.random.default_rng(case.seed * 7919 + 17 + seed_shift)
    out = {}
    for name in case.params:
        shape = PARAM_SHAPES[name[0]](rows, d, m)
        v = rng.uniform(-1.5, 1.5, size=shape)
        if rng.random() < 0.3:  # on a threshold now and then: comparisons see equality
            v = np.where(rng.random(shape) < 0.3, rng.choice(THRESHOLDS, size=shape), v)
        out[name] = v
    return out


def torch_params(case, rows, d, m, dtype, device, cpu_scalars):
    """The parameters as tensors of `dtype` on `device`; 'o*' sit one element into their storage, and with
    `cpu_scalars` the 0-d 'k*' are CPU tensors (immediates of the tape)."""
    out = {}
    for name, v in param_values(case, rows, d, m).items():
        if name[0] == 'o':
            store = torch.zeros(v.size + 1, dtype=dtype, device=device)
            store[1:] = torch.from_numpy(v.reshape(-1)).to(dtype=dtype, device=device)
            out[name] = store[1:].view(v.shape)
        elif name[0] == 'k':
            out[name] = torch.tensor(float(v), dtype=dtype, device='cpu' if cpu_scalars else device)
        else:
            out[name] = torch.from_numpy(v).to(dtype=dtype, device=device).contiguous()
    return out


def numpy_params(tparams, npt):
    return {k: v.cpu().numpy().astype(npt) for k, v in tparams.items()}


class FuzzSDE(nn.Module):
    """The case as an SDE on `device`: f and g run its statements with torch ops."""

    def __init__(self, case, sde_type, rows, d, m=None, dtype=torch.float32, device='cuda'):
        super().__init__()
        self.case, self.sde_type = case, sde_type
        self.noise_type = 'diagonal' if not case.general else 'additive' if case.layout == 'sra' else 'general'
        self.m = m or 1
        self.p = torch_params(case, rows, d, self.m, dtype, device, cpu_scalars=True)

    def f(self, t, y):
        return run_torch(self.case.f, self.case.f_out, t, y, self.p, self.m)

    def g(self, t, y):
        return run_torch(self.case.g, self.case.g_out, t, y, self.p, self.m)


# -- the generator ---------------------------------------------------------------------------------------------------
class _Value:
    __slots__ = ('shape', 'bool', 'bound', 'ydep', 'fresh', 'wide')

    def __init__(self, shape, boolean=False, bound=0.0, ydep=False, fresh=False, wide=False):
        self.shape, self.bool, self.bound, self.ydep, self.fresh, self.wide = shape, boolean, bound, ydep, fresh, wide


class _Gen:
    """Draws the statements of one callable."""

    def __init__(self, rng, params, prefix, rows, d, m, transcendental, inplace, sign, square, ydep=True):
        self.rng, self.prefix, self.rows, self.d, self.m = rng, prefix, rows, d, m
        self.tx, self.inplace, self.sign, self.square = transcendental, inplace, sign, square
        self.stmts, self.vals, self.n = [], {}, 0
        self.full = (rows, d)
        self.env = {'y': _Value(self.full, bound=YMAX, ydep=ydep), 't': _Value((), bound=1.0)}
        for name in params:
            shape = PARAM_SHAPES[name[0]](rows, d, m)
            self.env[name] = _Value(shape, bound=1.5, wide=name[0] in 'qwS')
        self.params = list(params)

    # values
    def _new(self, op, args, shape=None, boolean=False, bound=0.0, ydep=None, wide=None):
        names = [a for a in args if isinstance(a, str)]
        if names and all(a[0] == 'k' for a in names):  # (an op of CPU scalars alone would run on the CPU)
            args = tuple('s0' if a == names[0] else a for a in args)
        shape = shape or tuple(np.broadcast_shapes(*[self.env[a].shape for a in args if isinstance(a, str)]))
        if ydep is None:
            ydep = any(self.env[a].ydep for a in args if isinstance(a, str) and not self.env[a].bool)
        if wide is None:
            wide = any(self.env[a].wide for a in args if isinstance(a, str)) or len(shape) == 3
        name = f'{self.prefix}{self.n}'
        self.n += 1
        self.stmts.append((name, op, tuple(args)))
        self.env[name] = _Value(shape, boolean, bound, ydep, fresh=op not in ('lift', 'expand'), wide=wide)
        if not boolean and bound > BMAX and op != 'clamp':
            return self._new('clamp', (name, -BMAX, BMAX), bound=BMAX)
        return name

    def _floats(self, wide=None):
        return [k for k, v in self.env.items() if not v.bool and (wide is None or v.wide == wide or
                                                                    (wide and not v.wide and k == 't'))]

    def pick(self, pool, recent=0.6):
        """An operand: a recent value with probability `recent`, else anything in the pool."""
        made = [k for k in pool if k.startswith(self.prefix)]
        if made and self.rng.random() < recent:
            return made[-1 - int(self.rng.integers(0, min(4, len(made))))]
        return pool[int(self.rng.integers(0, len(pool)))]

    def number(self, table=NUMBERS):
        return float(table[int(self.rng.integers(0, len(table)))])

    def b(self, a):
        return self.env[a].bound if isinstance(a, str) else abs(a)

    def positive(self, x):
        """|x| + 1/2 (or x * x + 1/4): a value bounded away from zero."""
        if self.rng.random() < 0.7:
            ab = self._new('abs', (x,), bound=self.b(x))
            return self._new('add', (ab, 0.5), bound=self.b(x) + 0.5)
        sq = self._new('mul', (x, x), bound=self.b(x) ** 2)
        return self._new('add', (sq, 0.25), bound=self.b(sq) + 0.25)

    def mask(self, pool):
        """A comparison, sometimes compounded with &, | and ~; one time in three an earlier mask of this callable (of
        the pool's class, (rows, d) or per channel), so a SEL's condition stays live after it."""
        wide = any(self.env[v].wide for v in pool)
        masks = [k for k, v in self.env.items() if v.bool and k.startswith(self.prefix) and v.wide == wide]
        if masks and self.rng.random() < 1 / 3:
            return masks[int(self.rng.integers(0, len(masks)))]
        a = self.pick(pool)
        ops = ['lt', 'le', 'gt', 'ge', 'eq', 'ne']
        op = ops[int(self.rng.integers(0, len(ops)))]
        other = self.number(THRESHOLDS) if self.rng.random() < 0.5 else self.pick(pool, 0.3)
        c = self._new(op, (a, other), boolean=True)
        r = self.rng.random()
        if r < 0.25:
            c2 = self._new(ops[int(self.rng.integers(0, 6))], (self.pick(pool), self.number(THRESHOLDS)), boolean=True)
            c = self._new('and' if self.rng.random() < 0.5 else 'or', (c, c2), boolean=True)
        if self.rng.random() < 0.15:
            c = self._new('not', (c,), boolean=True)
        return c

    def op(self, pool):
        """One random op on operands of `pool` (names of float values); returns the new value's name."""
        rng, cat = self.rng, self.rng.random()
        a = self.pick(pool)
        if cat < 0.45:  # arithmetic
            kinds = ['mul', 'add', 'sub', 'rsub', 'nsub', 'div', 'divn', 'neg', 'sqrt'] + \
                ['sq'] * self.square + ['imul', 'iadd'] * self.inplace
            k = kinds[int(rng.integers(0, len(kinds)))]
            if k in ('imul', 'iadd'):
                targets = [v for v in pool if v.startswith(self.prefix) and self.env[v].fresh and
                           self.env[v].shape == self.full]
                if not targets:
                    k = 'mul'
                else:
                    a, other = targets[-1], self.pick(pool, 0.3)
                    if self.b(a) * max(self.b(other), 1.0) > BMAX or self.b(a) + self.b(other) > BMAX:
                        k, other = 'imul', self.number((0.5, 0.7, -0.25))
                    bound = self.b(a) * self.b(other) if k == 'imul' else self.b(a) + self.b(other)
                    name = self._new(k, (a, other), shape=self.full, bound=bound)
                    self.env[a] = self.env[name]
                    return name
            if k in ('mul', 'add', 'sub', 'rsub'):
                b = self.pick(pool, 0.3) if rng.random() < 0.75 else self.number()
                if k == 'rsub' and not isinstance(b, str):
                    k = 'nsub'
                bound = self.b(a) * self.b(b) if k == 'mul' else self.b(a) + self.b(b)
                return self._new(k, (a, b), bound=bound)
            if k == 'nsub':
                n = self.number()
                return self._new('nsub', (a, n), bound=self.b(a) + abs(n))
            if k == 'div':
                den = self.positive(self.pick(pool, 0.3))
                return self._new('div', (a, den), bound=2 * self.b(a))
            if k == 'divn':
                n = self.number(DIVISORS)
                return self._new('divn', (a, n), bound=self.b(a) / n)
            if k == 'neg':
                return self._new('neg', (a,), bound=self.b(a))
            if k == 'sqrt':
                x = self.positive(a)
                return self._new('sqrt', (x,), bound=math.sqrt(self.b(x)))
            return self._new('sq', (a,), bound=self.b(a) ** 2)
        if cat < 0.85 or not self.tx:  # comparison and selection
            kinds = ['clamp', 'clampmin', 'clampmax', 'clampt', 'clampmint', 'relu', 'abs', 'maximum', 'minimum',
                     'where', 'where', 'mfill', 'recip'] + ['sign'] * self.sign
            k = kinds[int(rng.integers(0, len(kinds)))]
            if k == 'clamp':
                lo = self.number((-1.0, -0.5, 0.0, 0.1))
                return self._new('clamp', (a, lo, lo + self.number((0.5, 1.0, 2.0))), bound=max(abs(lo), 3.0))
            if k in ('clampmin', 'clampmax'):
                n = self.number(THRESHOLDS)
                return self._new(k, (a, n), bound=max(self.b(a), abs(n)))
            if k in ('clampt', 'clampmint'):
                # (clamp's tensor bounds are not wrapped numbers: a CPU scalar there, or as x, is a device mismatch)
                pool = [v for v in pool if v[0] != 'k']
                a = 's0' if a[0] == 'k' else a
                lo = self.pick(pool, 0.2)
                if k == 'clampmint':
                    return self._new(k, (a, lo), bound=max(self.b(a), self.b(lo)))
                hi = self.pick(pool, 0.2)
                return self._new(k, (a, lo, hi), bound=max(self.b(lo), self.b(hi)))
            if k in ('relu', 'abs', 'sign'):
                return self._new(k, (a,), bound=1.0 if k == 'sign' else self.b(a))
            if k in ('maximum', 'minimum'):
                b = self.pick(pool, 0.3)
                return self._new(k, (a, b), bound=max(self.b(a), self.b(b)))
            if k == 'recip':
                x = self.positive(a)
                return self._new('recip', (x,), bound=2.0)
            c = self.mask(pool)
            if k == 'mfill' and a[0] != 'k' and \
                    np.broadcast_shapes(self.env[a].shape, self.env[c].shape) == self.env[a].shape:
                n = self.number()
                return self._new('mfill', (a, c, n), shape=self.env[a].shape, bound=max(self.b(a), abs(n)))
            b = self.pick(pool, 0.3) if rng.random() < 0.7 else self.number()
            return self._new('where', (c, a, b), bound=max(self.b(a), self.b(b)))
        # transcendental
        k = TRANSCENDENTAL[int(rng.integers(0, len(TRANSCENDENTAL)))]
        if k in ('exp', 'expm1'):
            x = self._new('clamp', (a, -3.0, 3.0), bound=3.0)
            return self._new(k, (x,), bound=math.exp(3.0))
        if k in ('log', 'rsqrt', 'log1p'):
            x = self.positive(a)
            return self._new(k, (x,), bound=max(2.0, math.log(self.b(x) + 1)) if k != 'rsqrt' else 1.5)
        if k == 'pow':
            x = self.positive(a)
            e = self.number(POWERS if self.square else tuple(p for p in POWERS if p != 2.0))
            return self._new('pow', (x, e), bound=max(self.b(x), 2.0) ** abs(e))
        return self._new(k, (a,), bound=1.0)


def _diag_callable(gen, n_ops, size, params, result_sel, ydep_result):
    """The statements of a (rows, d)-class callable: `n_ops` random ops, or for 'limits' a wide DAG."""
    pool = lambda: [k for k, v in gen.env.items() if not v.bool and not v.wide]  # noqa: E731
    if size == 'limits':
        # many values live at once, each reading its own parameter, then folded in an order of the draw
        row_like = [p for p in params if p[0] in 'cro' and not gen.env[p].wide]
        k = int(gen.rng.choice([14, 16, 17, 18, 19, 20, 22, 23, 24, 25]))
        live = []
        for i in range(k):
            src = row_like[i % len(row_like)] if row_like else gen.number()
            op = ('mul', 'sub', 'add')[i % 3]
            live.append(gen._new(op, ('y', src), bound=YMAX * 1.5 if op == 'mul' else YMAX + 1.5))
        gen.rng.shuffle(live)
        acc = live[0]
        for v in live[1:]:
            op = 'add' if gen.rng.random() < 0.6 else 'maximum'
            acc = gen._new(op, (acc, v), bound=gen.b(acc) + gen.b(v) if op == 'add' else max(gen.b(acc), gen.b(v)))
        out = acc
    else:
        out = 'y'
        for _ in range(n_ops):
            out = gen.op(pool())
    if result_sel and not gen.env[out].bool:
        c = gen.mask(pool())
        out = gen._new('where', (c, out, gen.pick(pool(), 0.3)), bound=BMAX)
    if gen.env[out].shape != gen.full or ydep_result and not gen.env[out].ydep:
        out = gen._new('mul' if gen.rng.random() < 0.5 else 'add', (out, 'y'), bound=gen.b(out) * YMAX + YMAX)
    return out


def _general_g(gen, n_ops, params, additive):
    """The statements of a (rows, d, m) g: a (rows, d)-class part lifted by unsqueeze(-1), then per-channel ops with
    (d, 1), (m,) and (d, m) parameters, expanded to (rows, d, m) when the result is narrower."""
    rows, d, m = gen.rows, gen.d, gen.m
    lifted = []
    if not additive:
        cur = 'y'
        for _ in range(max(1, n_ops // 3)):
            cur = gen.op([k for k, v in gen.env.items() if not v.bool and not v.wide])
        lifted.append(gen._new('lift', (cur,), shape=gen.env[cur].shape + (1,), bound=gen.b(cur), wide=True))
        if gen.rng.random() < 0.5:
            lifted.append(gen._new('lift', ('y',), shape=(rows, d, 1), bound=YMAX, wide=True))
    wide_params = [p for p in params if p[0] in 'qwS']
    pool = lambda: lifted + [k for k, v in gen.env.items() if v.wide and not v.bool and k not in lifted] + \
        [p for p in params if p[0] in 'sk'] + ['t']  # noqa: E731
    out = None
    if additive and gen.rng.random() < 0.2:
        S = [p for p in wide_params if p[0] == 'S']
        return gen._new('expand', (S[0],), shape=(rows, d, m), bound=1.5, wide=True)
    for _ in range(max(1, n_ops - n_ops // 3)):
        out = gen.op(pool())
    if out is None or not gen.env[out].wide:
        out = gen._new('mul', (out or 't', wide_params[int(gen.rng.integers(0, len(wide_params)))]),
                       bound=gen.b(out or 't') * 1.5)
    if gen.env[out].shape != (rows, d, m):
        shape = gen.env[out].shape
        if len(shape) == 3 and shape[0] == rows or not additive and gen.rng.random() < 0.5:
            S = [p for p in wide_params if p[0] == 'S'][0]
            out = gen._new('mul', (out, S), bound=gen.b(out) * 1.5)
        if gen.env[out].shape != (rows, d, m):
            out = gen._new('expand', (out,), shape=(rows, d, m), bound=gen.b(out), wide=True)
    return out


def _params(rng, size, general):
    if size == 'limits':
        n_c, n_r = int(rng.integers(6, 14)), int(rng.integers(4, 10))
    elif size == 'medium':
        n_c, n_r = int(rng.integers(1, 4)), int(rng.integers(0, 3))
    else:
        n_c, n_r = int(rng.integers(0, 3)), int(rng.integers(0, 2))
    names = ['s0', 'k0'] + [f'c{i}' for i in range(n_c)] + [f'r{i}' for i in range(n_r)] + ['o0']
    if general:
        names += ['q0', 'w0', 'S0'] + (['S1', 'q1'] if size != 'small' else [])
    return tuple(names)


def case(seed, layout, size=None, transcendental=None, row_params=True):
    """The fuzzed SDE of `seed` for `layout`: size class from the seed unless given; the transcendental ops in the
    compiled layouts for two seeds in five unless `transcendental` says otherwise.  Without `row_params`, no (rows, d)
    parameter: f and g then run on any block of rows (a row_split solve)."""
    rng = np.random.default_rng([seed, list(LAYOUTS).index(layout)])
    size = size or SIZES[int(rng.choice(4, p=[0.4, 0.3, 0.15, 0.15]))]
    recorder, pattern, compiled = LAYOUTS[layout]
    if transcendental is None:
        transcendental = compiled and rng.random() < 0.4
    general = recorder == 'general'
    params = tuple(p for p in _params(rng, size, general) if row_params or p[0] not in 'ro')
    n_ops = {'small': int(rng.integers(2, 7)), 'medium': int(rng.integers(8, 13)), 'limits': int(rng.integers(2, 7)),
             'edge': int(rng.integers(3, 12))}[size]
    # at the limits one callable (or, for the two-program tapes, both) is the wide one
    wide = {'f': size == 'limits', 'g': size == 'limits'}
    if size == 'limits':
        wide[str(rng.choice(['f', 'g'] + ([] if recorder == 'milstein' else ['both'])))[0]] = False
        if recorder == 'general':  # (g is per channel: f is the wide one)
            wide = {'f': True, 'g': False}
    kind = rng.random()
    # f
    fg = _Gen(rng, params, 'v', ROWS, D, M, transcendental, inplace=True, sign=True, square=True)
    if kind < 0.08:
        f, f_out = (), 'y'  # f is y
    else:
        f_out = _diag_callable(fg, n_ops, 'limits' if wide['f'] else 'small', params,
                               result_sel=rng.random() < 0.2, ydep_result=False)
        f = tuple(fg.stmts)
    # g
    milstein = recorder == 'milstein'
    gg = _Gen(rng, params, 'u', ROWS, D, M, transcendental, inplace=not milstein, sign=not milstein,
              square=not milstein)
    if general:
        g_out = _general_g(gg, max(n_ops, 3) if size != 'limits' or wide['f'] else 14, params,
                           additive=layout == 'sra')
        g = tuple(gg.stmts)
    elif 0.08 <= kind < 0.16 and f and not (milstein and not (_milstein_safe(f) and fg.env[f_out].ydep)):
        g, g_out = tuple((t.replace('v', 'u', 1), op, tuple(a.replace('v', 'u', 1) if isinstance(a, str) and
                                                            a.startswith('v') else a for a in args))
                         for t, op, args in f), f_out.replace('v', 'u', 1)  # g is f
    elif 0.16 <= kind < 0.22:
        g, g_out = (), 'y'  # g is y
    else:
        if 0.22 <= kind < 0.35 and f and not milstein:
            # g starts from f's first statements (shared sub-DAG), recomputed
            k = max(1, len(f) // 2)
            for tgt, op, args in f[:k]:
                gg._new(op, tuple(a.replace('v', 'u', 1) if isinstance(a, str) and a.startswith('v') else a
                                  for a in args), shape=fg.env[tgt].shape, boolean=fg.env[tgt].bool,
                        bound=min(fg.env[tgt].bound, BMAX))
        g_out = _diag_callable(gg, n_ops, 'limits' if wide['g'] else 'small', params,
                               result_sel=rng.random() < 0.2, ydep_result=milstein)
        g = tuple(gg.stmts)
    return Case(int(seed), layout, size, f, f_out, g, g_out, params, bool(transcendental))


def _milstein_safe(stmts):
    """Whether statements may serve as Milstein's g (autograd's vjp of them is a tape the recorder takes)."""
    return not any(op in ('sign', 'sq', 'imul', 'iadd') or op == 'pow' and args[1] == 2.0 for _, op, args in stmts)


def edge_state(rows, d, dtype, seed=0):
    """A y0 of the 'edge' class: 0, -0, negatives, every threshold and its neighbours, inf and NaN, shuffled."""
    npt = np.float32 if dtype == torch.float32 else np.float64
    vals = [0.0, -0.0, -1.0, 2.0, -3.5, np.inf, -np.inf, np.nan]
    for th in THRESHOLDS + (-0.25, 0.1, 0.3, 1.5):
        th = npt(th)
        vals += [th, np.nextafter(th, npt(np.inf)), np.nextafter(th, npt(-np.inf)), -th]
    vals = np.array(vals, dtype=npt)
    rng = np.random.default_rng(seed)
    out = vals[rng.integers(0, len(vals), size=rows * d)]
    out[:len(vals)] = vals[:rows * d]
    rng.shuffle(out)
    return torch.from_numpy(out.reshape(rows, d).copy())
