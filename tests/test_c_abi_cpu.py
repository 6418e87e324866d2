"""The ctypes binding (deva/_native.py) agrees with the C header (include/deva_b200.h): entry-point signatures, the
convolution descriptor's layout and the limits.  ctypes cannot see a prototype, so an argument list that drifts from
the header raises nothing at call time: the kernel receives garbage.  Parses the header only; no library, no GPU."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_C_KINDS = {'int': 'int32', 'int32_t': 'int32', 'int64_t': 'int64', 'size_t': 'uint64', 'uint64_t': 'uint64',
            'float': 'float'}
_CTYPES_KINDS = {ctypes.c_int32: 'int32', ctypes.c_int64: 'int64', ctypes.c_uint64: 'uint64', ctypes.c_size_t: 'uint64',
                 ctypes.c_float: 'float'}


def _header():
    text = open(os.path.join(ROOT, 'include', 'deva_b200.h')).read()
    text = re.sub(r'/\*.*?\*/', ' ', text, flags=re.S)
    return re.sub(r'//[^\n]*', ' ', text)


def _c_kind(decl):
    """Kind of the C type in a declaration: 'const float* qk', 'const float mean[3]', 'int64_t n', 'size_t'."""
    decl = ' '.join(decl.split())
    if '*' in decl or '[' in decl or 'deva_stream_t' in decl.split():
        return 'pointer'
    words = [w for w in decl.split() if w != 'const']
    assert words and words[0] in _C_KINDS, decl
    return _C_KINDS[words[0]]


def _ctypes_kind(t):
    if t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer):
        return 'pointer'
    return _CTYPES_KINDS[t]


def _prototypes():
    protos = {}
    for ret, name, params in re.findall(r'DEVA_B200_API\s+([^;()#]*?)\b(deva_b200_\w+)\s*\(([^)]*)\)\s*;', _header()):
        args = [] if params.strip() == 'void' else [_c_kind(p) for p in params.split(',')]
        protos[name] = (_c_kind(ret), args)
    return protos


def _conv_desc_fields():
    body = re.search(r'typedef\s+struct\s+deva_b200_conv_desc\s*\{(.*?)\}\s*deva_b200_conv_desc\s*;', _header(), re.S)
    fields = []
    for decl in filter(None, (d.strip() for d in body.group(1).split(';'))):
        first, *more = decl.split(',')  # 'int32_t batch, h, w, cin_pad'
        name = re.search(r'(\w+)\s*$', first).group(1)
        kind = _c_kind(first)
        fields.append((name, kind))
        for other in more:
            assert re.fullmatch(r'\s*\w+\s*', other), decl
            fields.append((other.strip(), kind))
    return fields


def test_signatures_match_header():
    from deva import _native
    protos = _prototypes()
    assert set(_native._SIGNATURES) == set(protos)
    for name, (res, args) in _native._SIGNATURES.items():
        assert (_ctypes_kind(res), [_ctypes_kind(a) for a in args]) == protos[name], name


def test_conv_desc_matches_header():
    from deva import _native
    fields = _conv_desc_fields()
    assert [(name, _ctypes_kind(t)) for name, t in _native.ConvDesc._fields_] == fields


def test_limits_match_header():
    from deva import _native
    macros = {k: int(v) for k, v in re.findall(r'#define\s+(DEVA_B200_\w+)\s+(\d+)\b', _header())}
    assert _native.ABI_VERSION == macros['DEVA_B200_ABI_VERSION']
    assert _native.LIST_PITCH == macros['DEVA_B200_LIST_PITCH']
    assert _native.MAX_GROUPS == macros['DEVA_B200_MAX_GROUPS']
    assert _native.MAX_SEGMENT_CHANNELS == macros['DEVA_B200_MAX_SEGMENT_CHANNELS']
