"""In-tree build of libstb200.so (the C-ABI CUDA library) with nvcc for sm_90a (H100).

The .so is a git-ignored build product next to this file; there is no JIT and no fallback: if the library is
missing, loading it raises.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / 'csrc'
INCLUDE = PKG_DIR.parent / 'include'
LIB_PATH = PKG_DIR / 'libstb200.so'
TEST_LIB_PATH = PKG_DIR / 'libstb200_test.so'   # product objects + csrc/api_test.cu (kernel-level test hooks)
TEST_ONLY_SOURCES = {'api_test.cu'}
OBJ_DIR = PKG_DIR / 'build'

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
    '-Xcompiler', '-fPIC', '-Xcompiler', '-fvisibility=hidden', '-cudart', 'static',
    f'-I{INCLUDE}', f'-I{CSRC}',
]


def _nvcc() -> str:
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not Path(nvcc).exists():
        raise RuntimeError('nvcc not found; libstb200.so cannot be built')
    return nvcc


def sources() -> list[Path]:
    return sorted(CSRC.glob('*.cu'))


def _stale() -> bool:
    if not LIB_PATH.exists() or not TEST_LIB_PATH.exists():
        return True
    t = min(LIB_PATH.stat().st_mtime, TEST_LIB_PATH.stat().st_mtime)
    deps = list(CSRC.glob('*')) + list(INCLUDE.glob('*.h')) + [Path(__file__)]
    return any(d.stat().st_mtime > t for d in deps)


def build_library(force: bool = False, verbose: bool = False) -> Path:
    """Compile every csrc/*.cu for sm_90a; link libstb200.so (product: everything but the test hooks) and
    libstb200_test.so (the same objects + api_test.o, loaded by tests/ only) next to this file."""
    if not force and not _stale():
        return LIB_PATH
    nvcc = _nvcc()
    OBJ_DIR.mkdir(exist_ok=True)

    def compile_one(src: Path) -> Path:
        obj = OBJ_DIR / (src.stem + '.o')
        hdr_t = max(p.stat().st_mtime for p in list(CSRC.glob('*.h')) + list(CSRC.glob('*.cuh')) +
                    list(INCLUDE.glob('*.h')) + [Path(__file__)])
        if not force and obj.exists() and obj.stat().st_mtime > max(src.stat().st_mtime, hdr_t):
            return obj
        cmd = [nvcc, *NVCC_FLAGS, '-c', str(src), '-o', str(obj)]
        if verbose:
            cmd.insert(1, '-Xptxas')
            cmd.insert(2, '-v')
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose:
            sys.stderr.write(r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f'nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}')
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        srcs = sources()
        objs = list(ex.map(compile_one, srcs))
    product = [o for o, src in zip(objs, srcs) if src.name not in TEST_ONLY_SOURCES]
    for target, members in ((LIB_PATH, product), (TEST_LIB_PATH, objs)):
        tmp = target.with_suffix('.so.tmp')
        cmd = [nvcc, '-shared', '-cudart', 'static', '-o', str(tmp), *map(str, members)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f'link failed:\n{r.stdout}\n{r.stderr}')
        os.replace(tmp, target)
    return LIB_PATH


if __name__ == '__main__':
    print(build_library(force='--force' in sys.argv, verbose='-v' in sys.argv))
