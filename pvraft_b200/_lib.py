"""ctypes binding of the C ABI, derived from its declarations in include/pvraft_b200.h.

The header is read at import: every `PVRAFT_API` function and every argument struct is bound from what the header says,
so the binding cannot drift from the declarations the library is compiled against.  This is not a C parser: after
comments and preprocessor lines are removed, the header may contain only these forms (anything else raises PvraftError
naming the declaration):
  - `PVRAFT_API <ret> pvraft_x(<params>);`  with <ret> one of int, int64_t, const char*, and `(void)` for no parameters;
  - `typedef struct pvraft_x { <fields> } pvraft_x;`  one or more `<type> <declarator>, ...;` per field line, a
    declarator optionally a fixed array (`const float* in[3];`);
  - `typedef enum pvraft_x { ... } pvraft_x;`  (not bound: the Python side names the values it uses);
  - the `extern "C" {` ... `}` wrapper.
Types: int, int64_t, float, double as scalars; pointers (const or not) to float, double, int32_t, int8_t, uint8_t,
uint16_t, int, void or one of the header's structs, all passed as c_void_p.  Each pointer's pointee is recorded
(FUNCTIONS, STRUCT_FIELDS) so that ops can check the tensor behind it.

The shared library is mandatory: importing the package never falls back to PyTorch ops or to the CPU oracle -- a
missing/unbuildable `libpvraft_b200.so` raises at first use.
"""
import ctypes as C
import keyword
import os
import re
import threading
from typing import NamedTuple

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libpvraft_b200.so')
HEADER_PATH = os.path.join(_HERE, '..', 'include', 'pvraft_b200.h')

IN_PLAIN, IN_GN, IN_GN_MINMAX = 0, 1, 2
ACT_NONE, ACT_RELU, ACT_LRELU = 0, 1, 2
KNN = 32
MOMENTS = 16


class PvraftError(RuntimeError):
    pass


class Decl(NamedTuple):
    """One parameter or struct field of the C ABI."""
    name: str          # as Python spells it (a keyword gets a trailing '_': `in` -> `in_`)
    ctype: object      # its ctypes type (an array type for a fixed array field)
    pointee: object    # the C type a pointer points to ('float', 'pvraft_linear_args', ...); None for a scalar
    length: int        # elements of a fixed array field; 1 otherwise


_SCALARS = {'int': C.c_int, 'int64_t': C.c_int64, 'float': C.c_float, 'double': C.c_double}
_POINTEES = {'float', 'double', 'int32_t', 'int8_t', 'uint8_t', 'uint16_t', 'int', 'void'}
_RETURNS = {'int': C.c_int, 'int64_t': C.c_int64, 'const char*': C.c_char_p}

_FORM = re.compile(r'''\s*(?:
    (?P<extern>extern\s+"C"\s*\{) | (?P<close>\}) |
    typedef\s+enum\s+(?P<enum>\w+)\s*\{[^{}]*\}\s*(?P=enum)\s*; |
    typedef\s+struct\s+(?P<struct>\w+)\s*\{(?P<fields>[^{}]*)\}\s*(?P=struct)\s*; |
    PVRAFT_API\s+(?P<ret>[\w\s*]*?)\s*\b(?P<fn>pvraft_\w+)\s*\((?P<params>[^()]*)\)\s*;
)''', re.X)
_TYPE = re.compile(r'\s*(?:const\s+)?(\w+)\s*(.*)', re.S)
_DECLARATOR = re.compile(r'\s*(\*?)\s*(\w+)\s*(?:\[(\d+)\])?\s*')


def _decls(text, structs, what, arrays):
    """`<type> <declarator>[, <declarator> ...]` -> [Decl]; `what` names the declaration in errors."""
    m = _TYPE.fullmatch(text)
    if not m:
        raise PvraftError(f'{HEADER_PATH}: cannot read `{text.strip()}` in {what}')
    base, out = m.group(1), []
    for d in m.group(2).split(','):
        dm = _DECLARATOR.fullmatch(d)
        if not dm or (dm.group(3) and not arrays):
            raise PvraftError(f'{HEADER_PATH}: cannot read `{text.strip()}` in {what}')
        star, name, length = dm.group(1), dm.group(2), int(dm.group(3) or 1)
        if star:
            if base not in _POINTEES and base not in structs:
                raise PvraftError(f'{HEADER_PATH}: pointer to unknown type `{base}` in {what}')
            ctype, pointee = C.c_void_p, base
        else:
            if base not in _SCALARS:
                raise PvraftError(f'{HEADER_PATH}: unknown type `{base}` in {what}')
            ctype, pointee = _SCALARS[base], None
        name = name + '_' if keyword.iskeyword(name) else name
        out.append(Decl(name, ctype * length if length > 1 else ctype, pointee, length))
    return out


def parse_header(text):
    """Header text -> (functions {name: (restype, [Decl])}, structs {name: [Decl]}), in declaration order."""
    text = re.sub(r'/\*.*?\*/', ' ', text, flags=re.S)      # a comment ends at its first */
    text = re.sub(r'^[ \t]*#.*$', ' ', text, flags=re.M)
    functions, structs = {}, {}
    pos = 0
    while text[pos:].strip():
        m = _FORM.match(text, pos)
        if not m:
            raise PvraftError(f'{HEADER_PATH}: unsupported declaration `{text[pos:].strip().splitlines()[0]}`')
        pos = m.end()
        if m.group('struct'):
            what = f'struct {m.group("struct")}'
            structs[m.group('struct')] = [d for line in m.group('fields').split(';') if line.strip()
                                          for d in _decls(line, structs, what, arrays=True)]
        elif m.group('fn'):
            name, ret, params = m.group('fn'), re.sub(r'\s*\*', '*', m.group('ret').strip()), m.group('params').strip()
            if ret not in _RETURNS:
                raise PvraftError(f'{HEADER_PATH}: unsupported return type `{ret}` of {name}')
            functions[name] = (_RETURNS[ret], [] if params == 'void' else
                               [d for p in params.split(',') for d in _decls(p, structs, name, arrays=False)])
    return functions, structs


def _class_name(struct):
    """pvraft_tc_linear_args -> TcLinearArgs; pvraft_corrfeat_args -> CorrFeatArgs, pvraft_flowout_args -> FlowOutArgs."""
    stem = struct[len('pvraft_'):-len('_args')]
    return {'corrfeat': 'CorrFeat', 'flowout': 'FlowOut'}.get(stem, stem.title().replace('_', '')) + 'Args'


with open(HEADER_PATH) as _f:
    FUNCTIONS, STRUCT_FIELDS = parse_header(_f.read())
# the argument structs as ctypes classes, by their C name and under their Python names (LinearArgs, TcLinearArgs, ...)
STRUCTS = {s: type(_class_name(s), (C.Structure,), {'_fields_': [(d.name, d.ctype) for d in fields]})
           for s, fields in STRUCT_FIELDS.items()}
globals().update({cls.__name__: cls for cls in STRUCTS.values()})
_SIGNATURES = {name: (res, [d.ctype for d in params]) for name, (res, params) in FUNCTIONS.items()}
EXPORTS = tuple(_SIGNATURES)

_lib = None
_lock = threading.Lock()


def lib():
    """The loaded shared library (built on first use if nvcc is available; otherwise an error)."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    from . import build as _build
                    try:
                        _build.build()
                    except Exception as e:   # noqa: BLE001
                        raise PvraftError(f'libpvraft_b200.so is missing and could not be built: {e}') from e
                handle = C.CDLL(LIB_PATH)
                for name, (res, args) in _SIGNATURES.items():
                    fn = getattr(handle, name)    # AttributeError => header/library mismatch: fail loudly
                    fn.restype = res
                    fn.argtypes = args
                _lib = handle
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().pvraft_last_error_string()
        raise PvraftError(f'{what} failed (code {rc}): {msg.decode() if msg else "?"}')
