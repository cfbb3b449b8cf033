"""ctypes binding of libptb_b200.so, derived from the C ABI's header include/ptb_b200.h.

The header is the one place that states a signature, a struct or a constant: on import this module parses its prototypes into
SIGNATURES, its two structs into RefineCfg and MatchCost, and its integer #defines into DEFINES, so the binding agrees with the
header by construction.  A type the parser does not know raises instead of being guessed.

There is NO fallback: if the CUDA library is missing or fails to load, every op raises.
"""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libptb_b200.so')
HEADER_PATH = os.path.normpath(os.path.join(_HERE, '..', 'include', 'ptb_b200.h'))

_lib = None
MISSING = []

# by-value C types of the ABI; every pointer is a c_void_p
_SCALARS = {'int': ctypes.c_int, 'int32_t': ctypes.c_int, 'int64_t': ctypes.c_int64, 'uint64_t': ctypes.c_uint64,
            'float': ctypes.c_float, 'double': ctypes.c_double}


def _struct_name(c_name):
    """ptb_refine_cfg -> RefineCfg"""
    return ''.join(w.capitalize() for w in c_name[len('ptb_'):].split('_'))


def parse_header(text):
    """(SIGNATURES, structs, defines) of a header's text: {name: (restype, argtypes)} of every ptb_* prototype,
    {C typedef name: ctypes.Structure subclass} and {PTB_*: int}.  Raises ValueError, naming the declaration, on a
    type or a statement it does not know."""
    defines = {m[1]: int(m[2]) for m in re.finditer(r'^\s*#\s*define\s+(PTB_\w+)\s+(-?\d+)\s*$', text, re.M)}
    src = re.sub(r'/\*.*?\*/', ' ', text, flags=re.S)
    src = re.sub(r'^\s*#.*$', '', src, flags=re.M)

    structs = {}
    for m in re.finditer(r'typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;', src, re.S):
        fields = []
        for member in filter(None, (s.strip() for s in m[1].split(';'))):
            f = re.fullmatch(r'(\w+)\s+(\w+(?:\s*,\s*\w+)*)', member)
            if f is None or f[1] not in _SCALARS:
                raise ValueError(f'struct {m[2]}: unknown member {member!r}')
            fields += [(n.strip(), _SCALARS[f[1]]) for n in f[2].split(',')]
        structs[m[2]] = type(_struct_name(m[2]), (ctypes.Structure,), {'_fields_': fields})
    src = re.sub(r'typedef\s+struct\s*\{.*?\}\s*\w+\s*;', '', src, flags=re.S)
    src = re.sub(r'extern\s+"C"\s*\{|\}', '', src)

    def ctype(t, decl, ret=False):
        t = ' '.join(t.replace('*', ' * ').split())
        if '*' in t:
            return ctypes.c_char_p if ret and t == 'const char *' else ctypes.c_void_p
        if t in _SCALARS:
            return _SCALARS[t]
        if t in structs and not ret:
            return structs[t]
        raise ValueError(f'unknown type {t!r} in {decl!r}')

    signatures = {}
    for decl in filter(None, (' '.join(s.split()) for s in src.split(';'))):
        m = re.fullmatch(r'(.+?)\b(ptb_\w+)\s*\((.*)\)', decl)
        if m is None:
            raise ValueError(f'not a ptb_* prototype: {decl!r}')
        params = [p.strip() for p in m[3].split(',')]
        if params == ['void']:
            params = []
        args = []
        for p in params:
            a = re.fullmatch(r'(.*?)\b\w+', p)           # the type, without the parameter's name
            if a is None or not a[1].strip():
                raise ValueError(f'unnamed parameter {p!r} in {decl!r}')
            args.append(ctype(a[1], decl))
        signatures[m[2]] = (ctype(m[1], decl, ret=True), args)
    return signatures, structs, defines


def _read_header():
    if not os.path.exists(HEADER_PATH):
        raise RuntimeError(f'{HEADER_PATH} is missing: the ctypes binding of libptb_b200.so is read from this C ABI header, which '
                           'ships with the repository')
    with open(HEADER_PATH) as f:
        return parse_header(f.read())


SIGNATURES, STRUCTS, DEFINES = _read_header()
RefineCfg = STRUCTS['ptb_refine_cfg']
MatchCost = STRUCTS['ptb_match_cost']


def load():
    """dlopen the in-tree library; raises (never falls back) when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f'{LIB_PATH} is missing: build it with `python -c "import __graft_entry__ as g; g.build()"` '
            '(nvcc, sm_90a). pointtinybenchmark_b200 has no CPU or PyTorch fallback.')
    lib = ctypes.CDLL(LIB_PATH)
    missing = []
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            missing.append(name)
            continue
        fn.restype = res
        fn.argtypes = args
    global MISSING
    MISSING = missing      # tests/test_capi_symbols.py requires this to be empty
    if lib.ptb_abi_version() != DEFINES['PTB_ABI_VERSION']:
        raise RuntimeError('libptb_b200.so ABI version mismatch')
    _lib = lib
    return lib


def check(rc, name):
    if rc != 0:
        msg = load().ptb_last_error().decode(errors='replace')
        raise RuntimeError(f'{name} failed (rc={rc}): {msg}')
