"""The stepper's C ABI for ctypes, read from its header `include/flybody_b200.h`, which states it once: prototypes, enums,
integer #defines and structs.  The reader knows the subset of C the header is written in and refuses anything else, naming the
line; it never guesses a type.  Prototypes take every pointer and FbHandle as c_void_p (`const char*`: c_char_p); struct fields
keep their pointee types.
"""
import ctypes as C
import functools
import os
import re
from types import SimpleNamespace

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'flybody_b200.h')

_SCALARS = {'int': C.c_int, 'int32_t': C.c_int32, 'uint8_t': C.c_uint8, 'uint32_t': C.c_uint32, 'uint64_t': C.c_uint64,
            'long long': C.c_longlong, 'float': C.c_float, 'double': C.c_double}
_TYPE = r'\s*(const\s+)?(long\s+long|\w+)\s*'          # a declaration's type: an optional const, then one word or `long long`
_STATEMENT = re.compile(r'''\s*(?:
    enum\s*(?P<enum>\w*)\s*\{(?P<items>[^}]*)\}\s*;
  | typedef\s+struct\s+\w+\s*\{(?P<fields>[^}]*)\}\s*(?P<struct>\w+)\s*;
  | typedef\s+struct\s+\w+\s*\*\s*(?P<handle>\w+)\s*;
  | (?P<ret>[^;(){}]+?)\b(?P<fn>\w+)\s*\((?P<params>[^()]*)\)\s*;
)''', re.X)


class StepperError(RuntimeError):
    pass


@functools.cache
def read(path=HEADER):
    """-> parse() of the header, read once per process"""
    if not os.path.exists(path):
        raise StepperError(f'stepper header not found at {path}: the package reads its C ABI from include/ beside it')
    with open(path) as f:
        return parse(f.read(), path)


def _parts(text, start, sep):
    """(offset, part) of every non-blank `sep`-separated part of text, which sits at offset `start`"""
    return [(start + p.start(), p[0].rstrip()) for p in re.finditer(rf'[^{sep}\s][^{sep}]*', text)]


def parse(text, path='<header>'):
    """-> namespace of functions {name: (restype, argtypes)}, enums {enum name: {enumerator: value}} (named enums), defines
    {name: int} and structs {typedef name: ctypes.Structure subclass}"""
    abi = SimpleNamespace(functions={}, enums={}, defines={}, structs={})
    handles = set()

    def fail(pos, what):
        line = text.count('\n', 0, pos) + 1
        raise StepperError(f'{path}:{line}: {what}: {text.splitlines()[line - 1].strip()!r}')

    def ctype(pos, decl, ret):
        """a return type (ret) or a named parameter of a prototype -> its ctypes type"""
        d = re.fullmatch(_TYPE + r'(\**)\s*(\w*)\s*', decl)
        if d and bool(d[4]) != ret:
            base, ptr = ' '.join(d[2].split()), d[3]
            if ptr == '*' and base == 'char' and d[1]:
                return C.c_char_p
            if base in handles or ptr and (base in _SCALARS or base in abi.structs or base in ('void', 'char')):
                return C.c_void_p
            if not ptr and (base in _SCALARS or ret and base == 'void'):
                return _SCALARS.get(base)                # void: None
        fail(pos, 'a type the reader does not know')

    # comments become blanks and preprocessor lines blank lines, so that offsets keep their lines
    lines = re.sub(r'/\*.*?\*/', lambda c: re.sub(r'\S', ' ', c[0]), text, flags=re.S).split('\n')
    cplusplus, off = False, 0
    for i, s in enumerate(lines):
        if cplusplus or s.lstrip().startswith('#'):
            s, lines[i] = s.strip(), ' ' * len(s)
            if cplusplus:                                # C++ only (extern "C"): the ABI is the C one
                cplusplus = s != '#endif'
            elif s == '#ifdef __cplusplus':
                cplusplus = True
            elif d := re.fullmatch(r'#define\s+(\w+)\s+(\d+)', s):
                abi.defines[d[1]] = int(d[2])
            elif not re.fullmatch(r'#(?:ifndef\s+\w+|define\s+\w+|include\s+<\w+\.h>|endif)', s):
                fail(off, 'a preprocessor line the reader does not know')
        off += len(lines[i]) + 1
    body, pos = '\n'.join(lines), 0
    while body[pos:].strip():
        m = _STATEMENT.match(body, pos)
        if not m:
            fail(pos + len(body[pos:]) - len(body[pos:].lstrip()), 'a construct the reader does not know')
        pos = m.end()
        if m['items'] is not None:
            values = {}
            for p, item in _parts(m['items'], m.start('items'), ','):
                if not (e := re.fullmatch(r'(\w+)\s*=\s*(-?\d+)', item)):
                    fail(p, 'an enumerator without an integer value')
                values[e[1]] = int(e[2])
            if m['enum']:
                abi.enums[m['enum']] = values
        elif m['fields'] is not None:
            fields = []
            for p, decl in _parts(m['fields'], m.start('fields'), ';'):
                d = re.fullmatch(_TYPE + r'(.*)', decl, re.S)
                base = d and _SCALARS.get(' '.join(d[2].split()))
                if base is None:
                    fail(p, 'a field type the reader does not know')
                for q, dcl in _parts(d[3], p + d.start(3), ','):
                    if not (v := re.fullmatch(r'(\*?)\s*(\w+)\s*((?:\[\s*\d+\s*\]\s*)*)', dcl)):
                        fail(q, 'a declarator the reader does not know')
                    t = C.POINTER(base) if v[1] else base
                    for n in reversed(re.findall(r'\d+', v[3])):
                        t = t * int(n)
                    fields.append((v[2], t))
            abi.structs[m['struct']] = type(m['struct'], (C.Structure,), {'_fields_': fields})
        elif m['handle']:
            handles.add(m['handle'])
        else:
            if not m['params'].strip():
                fail(m.start('fn'), 'a prototype without a parameter list (write `(void)`)')
            params = [] if m['params'].strip() == 'void' else _parts(m['params'], m.start('params'), ',')
            abi.functions[m['fn']] = (ctype(m.start('ret'), m['ret'], True), [ctype(p, a, False) for p, a in params])
    return abi
