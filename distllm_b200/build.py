"""In-tree build of the native library (libb2e.so) with nvcc for sm_90a.

nvcc cross-compiles without a GPU, so this runs on the authoring box too; the built .so sits next
to the package (git-ignored) and travels with the tree.
"""

from __future__ import annotations

import fcntl
import hashlib
import os
import shutil
import subprocess
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / 'csrc'
LIB_PATH = PKG_DIR / 'libb2e.so'             # 16-bit storage = IEEE half
LIB_PATH_BF16 = PKG_DIR / 'libb2e_bf16.so'    # the same sources with -DB2E_STORAGE_BF16 (storage = bfloat16)
LIBS = {'f16': (LIB_PATH, []), 'bf16': (LIB_PATH_BF16, ['-DB2E_STORAGE_BF16'])}
LOCK_PATH = PKG_DIR / '.build.lock'

NVCC_FLAGS = [
    '-O3',
    '-std=c++17',
    '-gencode',
    'arch=compute_90a,code=sm_90a',
    '-lineinfo',
    '-Xcompiler',
    '-fPIC',
    '-shared',
]


def _nvcc() -> str:
    exe = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not Path(exe).exists():
        raise RuntimeError('nvcc not found; cannot build libb2e.so')
    return exe


def sources() -> list[Path]:
    return sorted(CSRC.glob('*.cu')) + sorted(CSRC.glob('*.cuh')) + [
        PKG_DIR.parent / 'include' / 'b2e.h',
        PKG_DIR.parent / 'include' / 'b2e_debug.h',
    ]


def source_hash() -> str:
    h = hashlib.sha256(' '.join(NVCC_FLAGS).encode())
    for src in sources():
        h.update(src.name.encode())
        h.update(src.read_bytes())
    return h.hexdigest()


def _stamp(lib: Path) -> Path:
    return lib.with_name(lib.name + '.srchash')   # content hash of the sources the .so was built from


def is_stale(lib: Path = LIB_PATH) -> bool:
    """Content-based (a snapshot copied to another box need not keep mtimes)."""
    stamp = _stamp(lib)
    if not lib.exists() or not stamp.exists():
        return True
    return stamp.read_text().strip() != source_hash()


def _compile(lib: Path, defines: list[str], verbose: bool) -> subprocess.Popen:
    tmp = f'{lib}.{os.getpid()}.tmp'
    cmd = [_nvcc(), *NVCC_FLAGS, *defines, '-o', tmp, str(CSRC / 'b2e_api.cu')]
    if verbose:
        cmd[1:1] = ['-Xptxas', '-v']
    return subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)


def build_native(force: bool = False, verbose: bool = False) -> Path:
    """Compile csrc/b2e_api.cu into libb2e.so (half storage) and libb2e_bf16.so (bfloat16 storage), both nvcc
    runs side by side; skipped when up to date.  Safe to call from several ranks at once: one builds under a
    file lock, the others wait and find the result."""
    todo = [k for k, (lib, _) in LIBS.items() if force or is_stale(lib)]
    if not todo:
        return LIB_PATH
    with open(LOCK_PATH, 'w') as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            todo = [k for k, (lib, _) in LIBS.items() if force or is_stale(lib)]
            digest = source_hash()
            procs = {k: _compile(LIBS[k][0], LIBS[k][1], verbose) for k in todo}
            for k, proc in procs.items():
                out, err = proc.communicate()
                lib = LIBS[k][0]
                if proc.returncode != 0:
                    raise RuntimeError(f'nvcc failed ({lib.name}):\n{out}\n{err}')
                os.replace(f'{lib}.{os.getpid()}.tmp', lib)
                _stamp(lib).write_text(digest + '\n')
                if verbose:
                    print(err)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB_PATH


if __name__ == '__main__':
    print(build_native(force=True, verbose=True))
