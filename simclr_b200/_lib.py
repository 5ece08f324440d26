"""ctypes binding of libsimclr_b200.so, generated from include/simclr_b200.h.

There is no fallback: if the shared library is missing or a call fails, this
module raises.  `lib.<name>(...)` takes raw integers / floats / torch tensors
(tensors are passed as `data_ptr()`), checks the status code and raises
`SimclrError` carrying `simclr_last_error()`.
"""
import ctypes
import os
import re

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, '..', 'include', 'simclr_b200.h')
LIB_PATH = os.environ.get('SIMCLR_B200_LIB') or os.path.join(HERE, 'libsimclr_b200.so')   # override: A/B builds

F32, BF16 = 0, 1
DTYPE_CODE = {torch.float32: F32, torch.bfloat16: BF16}


class SimclrError(RuntimeError):
    pass


_CTYPES = {
    'int': ctypes.c_int, 'int64_t': ctypes.c_int64, 'float': ctypes.c_float, 'double': ctypes.c_double,
    'size_t': ctypes.c_size_t,
}


def parse_header(path=HEADER):
    """Returns {name: (restype, [(ctype, argname), ...])} for every SIMCLR_API declaration."""
    src = open(path).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    decls = {}
    for m in re.finditer(r'SIMCLR_API\s+([\w\s\*]+?)\s*\b(simclr_\w+)\s*\((.*?)\)\s*;', src, flags=re.S):
        ret, name, args = m.group(1).strip(), m.group(2), m.group(3).strip()
        if ret == 'int':
            restype = ctypes.c_int
        elif ret == 'size_t':
            restype = ctypes.c_size_t
        elif ret.replace(' ', '') == 'constchar*':
            restype = ctypes.c_char_p
        else:
            raise ValueError('unknown return type %r for %s' % (ret, name))
        argl = []
        if args and args != 'void':
            for a in args.split(','):
                a = a.strip()
                if '*' in a:
                    argl.append((ctypes.c_void_p, a.split('*')[-1].strip()))
                else:
                    toks = a.replace('const ', '').split()
                    argl.append((_CTYPES[toks[0]], toks[-1]))
        decls[name] = (restype, argl)
    return decls


def _conv(v, ct):
    if ct is ctypes.c_void_p:
        if v is None:
            return None
        if isinstance(v, torch.Tensor):
            return v.data_ptr()
        return int(v)
    return v


# kernels launched per C-ABI call (for the `gpu_launches` claim of bench.py)
_LAUNCHES = {'ntxent_forward': 3, 'ntxent_backward': 2, 'contrast_metrics': 3, 'softmax_xent': 2, 'l2_loss': 2,
             'lars_apply': 2, 'bn_bwd_apply': 2, 'version': 0, 'last_error': 0, 'ntxent_workspace_bytes': 0,
             'set_accumulate_prezeroed': 0, 'set_tc_multicast': 0, 'tc_max_active_clusters': 0, 'memset_zero': 0, 'conv2d_fprop_tc3': 6, 'conv2d_dgrad_tc3': 6, 'conv2d_wgrad_tc3': 6,
             'jpeg_decode': 3, 'distill_xent': 3, 'gcl_workspace_bytes': 0, 'gcl_lse_forward': 3,
             'gcl_lse_backward': 2, 'gcl_swd_forward': 5, 'gcl_swd_backward': 2}


class _Lib:
    def __init__(self):
        self._dll = None
        self._decls = parse_header()
        self.launch_count = 0

    def load(self):
        if self._dll is not None:
            return self
        if not os.path.exists(LIB_PATH):
            raise SimclrError(
                'libsimclr_b200.so not found at %s; run `python -m simclr_b200.build` '
                '(there is no CPU / PyTorch fallback for the hot path)' % LIB_PATH)
        self._dll = ctypes.CDLL(LIB_PATH)
        for name, (restype, argl) in self._decls.items():
            fn = getattr(self._dll, name)          # AttributeError if the symbol is not exported
            fn.restype = restype
            fn.argtypes = [ct for ct, _ in argl]
        return self

    @property
    def declarations(self):
        return self._decls

    def last_error(self):
        self.load()
        return self._dll.simclr_last_error().decode()

    def __getattr__(self, name):
        if name.startswith('_'):
            raise AttributeError(name)
        full = 'simclr_' + name
        if full not in self._decls:
            raise AttributeError(name)
        self.load()
        fn = getattr(self._dll, full)
        restype, argl = self._decls[full]
        cts = [ct for ct, _ in argl]
        nlaunch = _LAUNCHES.get(name, 1)

        def call(*args):
            if len(args) != len(cts):
                raise TypeError('%s expects %d arguments, got %d' % (full, len(cts), len(args)))
            r = fn(*[_conv(a, ct) for a, ct in zip(args, cts)])
            self.launch_count += nlaunch
            if restype is ctypes.c_int and name not in ('version', 'set_accumulate_prezeroed', 'set_tc_multicast',
                                                        'tc_max_active_clusters'):
                if r != 0:
                    raise SimclrError('%s failed with status %d: %s' % (full, r, self._dll.simclr_last_error().decode()))
                return None
            return r

        call.__name__ = full
        setattr(self, name, call)
        return call


lib = _Lib()


def stream_ptr():
    """The current torch CUDA stream as a raw cudaStream_t."""
    return torch.cuda.current_stream().cuda_stream
