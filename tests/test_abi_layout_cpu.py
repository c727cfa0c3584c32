"""CPU test: the package's ctypes statement of the C ABI agrees with include/orb_b200.h.  Every struct mirror has the header's size, field
names, order and offsets as gcc lays the header out, and every entry of SIGNATURES has the header's parameter and return kinds.  Needs
neither a GPU nor the built library."""
import ast
import ctypes as C
import glob
import keyword
import os
import re
import subprocess

import orb_slam3_modified_b200 as orb
from test_abi_cpu import _declared

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'orb_slam3_modified_b200')

# header scalar types -> the one ctypes type that passes them (c_int32 is c_int; size_t and uint64_t are both c_ulong on LP64)
ARG_KINDS = {'int': C.c_int, 'int32_t': C.c_int, 'float': C.c_float, 'double': C.c_double, 'size_t': C.c_size_t, 'uint64_t': C.c_uint64}
RET_KINDS = {'int': C.c_int, 'void': None, 'const char*': C.c_char_p}


def _header():
    """include/orb_b200.h without comments and preprocessor lines."""
    src = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'orb_b200.h')).read(), flags=re.S)
    return re.sub(r'^[ \t]*#.*$', '', src, flags=re.M)


def _header_structs():
    """{typedef name: field names in declaration order} of the header's structs."""
    out = {}
    for body, name in re.findall(r'typedef\s+struct\s+\w+\s*\{(.*?)\}\s*(\w+)\s*;', _header(), flags=re.S):
        decls = [d for d in body.split(';') if d.strip()]
        out[name] = [re.search(r'(\w+)\s*(?:\[[^\]]*\])?\s*$', part).group(1) for d in decls for part in d.split(',')]
    return out


def _header_prototypes():
    """{function: (return type, [parameter kinds])}, a kind being 'pointer' or the scalar type without const and the parameter name."""
    out = {}
    for ret, name, params in re.findall(r'(?<=[;{}])\s*((?:const\s+)?\w+\s*\**)\s*(\w+)\s*\(([^()]*)\)\s*;', _header()):
        kinds = []
        for p in params.split(','):
            words = [w for w in p.split() if w != 'const']
            if words != ['void']:
                kinds.append('pointer' if '*' in p else ' '.join(words[:-1]))
        out[name] = (re.sub(r'\s*\*', '*', ' '.join(ret.split())), kinds)
    return out


def _mirrors():
    """{header struct: ctypes class or numpy dtype} of the package's mirrors; a class is named after its struct, '_' prefix optional."""
    m = {n.lstrip('_'): v for n, v in vars(orb).items() if isinstance(v, type) and issubclass(v, C.Structure)}
    m.update(OrbKeyPoint=orb.KP_DTYPE, OrbmNewPoint=orb.NEW_POINT_DTYPE)
    return m


def _python_layout(mirror):
    """(size, [(field, offset)]) of a ctypes class or numpy dtype; a keyword field's trailing '_' is dropped (LbaResult.lambda_)."""
    plain = lambda n: n[:-1] if n.endswith('_') and keyword.iskeyword(n[:-1]) else n
    if isinstance(mirror, type):
        return C.sizeof(mirror), [(plain(f[0]), getattr(mirror, f[0]).offset) for f in mirror._fields_]
    return mirror.itemsize, [(n, mirror.fields[n][1]) for n in mirror.names]


def _gcc_layout(tmp_path, structs):
    """{struct: (sizeof, [(field, offsetof)])} as gcc lays out the header, for the named structs with the header's own field lists."""
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "orb_b200.h"', 'int main(void) {']
    for s, fields in structs.items():
        lines.append('    printf("%%s %%zu", "%s", sizeof(%s));' % (s, s))
        lines += ['    printf(" %%zu", offsetof(%s, %s));' % (s, f) for f in fields]
        lines.append('    printf("\\n");')
    lines += ['    return 0;', '}']
    (tmp_path / 'layout.c').write_text('\n'.join(lines) + '\n')
    exe = str(tmp_path / 'layout')
    subprocess.run(['gcc', '-std=c11', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(tmp_path / 'layout.c'), '-o', exe], check=True)
    out = {}
    for row in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split('\n'):
        if row:
            name, size, *offs = row.split()
            out[name] = (int(size), list(zip(structs[name], map(int, offs))))
    return out


def test_struct_mirrors_match_header_layout(tmp_path):
    mirrors, header = _mirrors(), _header_structs()
    assert len(mirrors) >= 25 and set(mirrors) <= set(header), sorted(set(mirrors) - set(header))
    gcc = _gcc_layout(tmp_path, {s: header[s] for s in mirrors})
    for s, mirror in sorted(mirrors.items()):
        size, fields = _python_layout(mirror)
        assert [f for f, _ in fields] == header[s], (s, 'field names / order')
        assert fields == gcc[s][1], (s, 'offsets', [(p, g) for p, g in zip(fields, gcc[s][1]) if p != g])
        assert size == gcc[s][0], (s, 'sizeof', size, gcc[s][0])


def test_structure_classes_only_at_module_level():
    """One mirror per struct: no ctypes Structure is declared inside a function or another class of the package."""
    for path in glob.glob(os.path.join(PKG, '*.py')):
        tree = ast.parse(open(path).read())
        top = {id(n) for n in tree.body}
        nested = [n.name for n in ast.walk(tree) if isinstance(n, ast.ClassDef) and id(n) not in top
                  and any(isinstance(b, ast.Attribute) and b.attr == 'Structure' for b in n.bases)]
        assert not nested, (path, nested)


def test_signatures_match_header_prototypes():
    protos = _header_prototypes()
    assert sorted(protos) == _declared()        # the same declarations test_abi_cpu checks the library's exports against
    for name, (restype, argtypes) in orb.SIGNATURES.items():
        assert name in protos, name
        ret, kinds = protos[name]
        assert restype is RET_KINDS[ret], (name, 'return', ret, restype)
        assert len(argtypes) == len(kinds), (name, 'parameter count', len(argtypes), len(kinds))
        for k, (kind, t) in enumerate(zip(kinds, argtypes)):
            if kind == 'pointer':
                assert t is C.c_void_p or issubclass(t, C._Pointer), (name, k, kind, t)
            else:
                assert t is ARG_KINDS[kind], (name, k, kind, t)


def test_every_header_function_the_package_names_has_a_signature():
    src = '\n'.join(open(p).read() for p in glob.glob(os.path.join(PKG, '*.py')))
    named = [n for n in _header_prototypes() if re.search(r'\b%s\b' % n, src)]
    assert len(named) >= 60
    assert not [n for n in named if n not in orb.SIGNATURES]
