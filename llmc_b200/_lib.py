"""ctypes binding of libllmc_b200.so.

include/llmc_b200.h is the only statement of the C ABI: at import this module reads the header and
derives from it every entry point's restype and argtypes (SIGNATURES) and the enum / #define
constants (F32, OUT_*, MOE_MAX_EXPERTS, ...), so a signature is written once, in C.

There is deliberately NO CPU / eager fallback: if the CUDA library is missing or a kernel
reports an error the call raises.  (The oracle under oracle/ is test infrastructure and is
never imported from here.)
"""
import ctypes
import os
import re
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libllmc_b200.so')
HEADER_PATH = os.path.join(_HERE, '..', 'include', 'llmc_b200.h')


class LlmcB200Error(RuntimeError):
    pass


# every pointer binds as c_void_p, a `const char*` return value as c_char_p, these by name; any
# other C type is an error, never a default
_CTYPES = {'int': ctypes.c_int, 'int64_t': ctypes.c_int64, 'long long': ctypes.c_longlong,
           'float': ctypes.c_float, 'double': ctypes.c_double}


def _ctype(decl, proto):
    """ctypes class of the C type `decl` ('int64_t', 'const void * const *', ...) of prototype `proto`."""
    if '*' in decl:
        return ctypes.c_void_p
    if decl not in _CTYPES:
        raise LlmcB200Error(f'llmc_b200.h: {proto}: no ctypes binding for the C type {decl!r}')
    return _CTYPES[decl]


def parse_header(text):
    """(signatures, constants) of the C header `text`.  signatures: every prototype
    `ret llmc_*(params);` (the return type on the name's line, the parameters on any number of
    lines) as name -> (restype, [argtypes]); constants: every enum member with an explicit value
    and every integer `#define LLMC_*`, as name -> int."""
    text = re.sub(r'/\*.*?\*/', ' ', text, flags=re.S)
    consts = {n: int(v, 0) for n, v in re.findall(r'^[ \t]*#[ \t]*define[ \t]+(LLMC_\w+)[ \t]+(-?\d\w*)[ \t]*$',
                                                  text, flags=re.M)}
    for body in re.findall(r'\benum\s*\{(.*?)\}', text, flags=re.S):
        consts.update((n, int(v, 0)) for n, v in re.findall(r'\b(LLMC_\w+)\s*=\s*(-?\d\w*)', body))
    sigs = {}
    for ret, name, params in re.findall(r'^[ \t]*(\w[\w \t]*?\**)[ \t]*\b(llmc_\w+)\s*\(([^()]*)\)\s*;',
                                        text, flags=re.M):
        ret = ' '.join(ret.replace('*', ' *').split())
        params = [' '.join(p.split()) for p in params.split(',')]
        # a parameter is `type name`: drop the name unless the type is a pointer (which binds whole)
        sigs[name] = (ctypes.c_char_p if ret == 'const char *' else _ctype(ret, name),
                      [] if params == ['void'] else
                      [_ctype(p if '*' in p else p.rsplit(' ', 1)[0], name) for p in params])
    return sigs, consts


if not os.path.exists(HEADER_PATH):
    raise LlmcB200Error(f'{HEADER_PATH} not found: the ctypes bindings are read from this C header, '
                        'which sits in include/ beside the llmc_b200 package')
with open(HEADER_PATH) as _fh:
    SIGNATURES, CONSTANTS = parse_header(_fh.read())

F32, F16, BF16 = CONSTANTS['LLMC_F32'], CONSTANTS['LLMC_F16'], CONSTANTS['LLMC_BF16']
OUT_NONE, OUT_QDQ, OUT_CODES_I8, OUT_CODES_U8, OUT_CODES_I32, OUT_PACK_VLLM, OUT_FLAG_ZP_INSIDE = (
    CONSTANTS['LLMC_OUT_' + n] for n in ('NONE', 'QDQ', 'CODES_I8', 'CODES_U8', 'CODES_I32', 'PACK_VLLM',
                                         'FLAG_ZP_INSIDE'))
MOE_MAX_EXPERTS = CONSTANTS['LLMC_MOE_MAX_EXPERTS']

_DTYPE = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}

_lock = threading.Lock()
_lib = None


def load():
    """Load (once) and return the ctypes handle.  Raises if the library is missing."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise LlmcB200Error(
                f'{LIB_PATH} not found: build it with `python -m llmc_b200.build` '
                '(or __graft_entry__.build()).  llmc_b200 has no CPU fallback.')
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            try:
                fn = getattr(lib, name)
            except AttributeError:
                continue  # tests/test_abi.py reports missing symbols explicitly
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def dtype_enum(dt):
    try:
        return _DTYPE[dt]
    except KeyError:
        raise LlmcB200Error(f'unsupported dtype {dt}') from None


def ptr(t):
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())


def stream_ptr(device=None):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise LlmcB200Error(
                'llmc_b200 kernels run on CUDA tensors only (got a %s tensor); there is no CPU '
                'fallback in the product path' % t.device.type)


def check(rc, what):
    if rc != 0:
        lib = load()
        raise LlmcB200Error('%s failed: %s (%s)' % (
            what, lib.llmc_b200_error_string(rc).decode(), lib.llmc_b200_last_error().decode()))


def call(name, *args):
    lib = load()
    rc = getattr(lib, name)(*args)
    check(rc, name)
