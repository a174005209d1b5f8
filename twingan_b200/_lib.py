"""ctypes binding of libtwg.so (the C-ABI declared in include/twg.h, the JPEG decoder's in include/twgjpeg.h, the
progressive JPEG decoder's in include/twgjpegp.h, the JPEG encoder's in include/twgjenc.h and the PNG decoder's in
include/twgpng.h).

The prototypes are parsed from the header itself so the Python side can never drift from the ABI.
There is no CPU fallback: if the library is missing, or a kernel entry point is called without a CUDA
device, this module raises.
"""
from __future__ import annotations

import ctypes
import os
import re
from typing import Dict, List, Tuple

_HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'twg.h')
JPEG_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'twgjpeg.h')
JPEG_PREFIX = 'twgjpeg_'
JPEGP_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'twgjpegp.h')
JPEGP_PREFIX = 'twgjpegp_'
JENC_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'twgjenc.h')
JENC_PREFIX = 'twgjenc_'
PNG_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'twgpng.h')
PNG_PREFIX = 'twgpng_'
LIB_PATH = os.environ.get('TWG_LIB') or os.path.join(_HERE, 'libtwg.so')   # TWG_LIB: A/B builds of the same ABI

_CTYPES = {
    'const float*': ctypes.c_void_p, 'float*': ctypes.c_void_p, 'void*': ctypes.c_void_p,
    'const void*': ctypes.c_void_p, 'const int64_t*': ctypes.c_void_p, 'twg_stream_t': ctypes.c_void_p,
    'int': ctypes.c_int, 'int64_t': ctypes.c_int64, 'float': ctypes.c_float,
    'const char*': ctypes.c_char_p, 'void': None,
}


def parse_header(path: str = HEADER, prefix: str = 'twg_') -> Dict[str, Tuple[str, List[str]]]:
  """Returns {symbol: (return type, [arg types])} for every function named `prefix`* declared in the header (twg.h)."""
  src = open(path).read()
  src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
  src = re.sub(r'//[^\n]*', '', src)
  src = '\n'.join(l for l in src.splitlines() if not l.strip().startswith('#'))
  protos = {}
  for m in re.finditer(r'(const char\*|int64_t|int|void)\s+(' + re.escape(prefix) + r'\w+)\s*\(([^)]*)\)\s*;', src):
    ret, name, args = m.group(1), m.group(2), m.group(3).strip()
    types: List[str] = []
    if args and args != 'void':
      for a in args.split(','):
        a = ' '.join(a.split())
        t = re.sub(r'\s*\w+$', '', a) if not a.endswith('*') else a
        t = t.replace(' *', '*')
        types.append(t)
    protos[name] = (ret, types)
  return protos


class TwgError(RuntimeError):
  pass


class _Lib:
  def __init__(self):
    if not os.path.exists(LIB_PATH):
      raise TwgError('libtwg.so not built: run `python -c "import __graft_entry__ as g; g.build()"` '
                     '(there is no CPU fallback)')
    self.cdll = ctypes.CDLL(LIB_PATH)
    self.protos = parse_header()
    self.jpeg_protos = parse_header(JPEG_HEADER, JPEG_PREFIX)
    self.jpegp_protos = parse_header(JPEGP_HEADER, JPEGP_PREFIX)
    self.jenc_protos = parse_header(JENC_HEADER, JENC_PREFIX)
    self.png_protos = parse_header(PNG_HEADER, PNG_PREFIX)
    for name, (ret, args) in (list(self.protos.items()) + list(self.jpeg_protos.items())
                              + list(self.jpegp_protos.items()) + list(self.jenc_protos.items())
                              + list(self.png_protos.items())):
      fn = getattr(self.cdll, name)  # raises AttributeError if the symbol is not exported
      fn.restype = _CTYPES[ret]
      fn.argtypes = [_CTYPES[a] for a in args]

  def call(self, name: str, *args):
    rc = getattr(self.cdll, name)(*args)
    if rc != 0:
      raise TwgError('%s failed (%d): %s' % (name, rc, self.cdll.twg_last_error().decode()))

  def try_call(self, name: str, *args) -> int:
    return getattr(self.cdll, name)(*args)

  def last_error(self) -> str:
    return self.cdll.twg_last_error().decode()

  def launch_count(self) -> int:
    return int(self.cdll.twg_launch_count())


_LIB = None


def lib() -> _Lib:
  global _LIB
  if _LIB is None:
    _LIB = _Lib()
  return _LIB
