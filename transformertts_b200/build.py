"""Build libttsb.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m transformertts_b200.build [--force]

nvcc cross-compiles without a GPU; the resulting transformertts_b200/libttsb.so is git-ignored but travels to the
GPU box with the working-tree snapshot.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / 'csrc'
INCLUDE = PKG.parent / 'include'
OUT = PKG / 'libttsb.so'
OBJ_DIR = PKG / 'build'
SOURCES = ['host.cu', 'gemm_tc.cu', 'attention_tc.cu', 'bgemm_tc.cu', 'attn_probs_tc.cu', 'rowops.cu', 'stft_mel.cu', 'train_ops.cu', 'alignment.cu', 'dp_nccl.cu', 'griffin_lim.cu', 'decode.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC', '-Xcompiler', '-fvisibility=default', '--expt-relaxed-constexpr']


def _nvcc() -> str:
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (Path(cand).exists() or cand == 'nvcc'):
            return cand
    raise RuntimeError('nvcc not found')


def _digest() -> str:
    h = hashlib.sha256()
    for f in sorted(list(CSRC.glob('*')) + [INCLUDE / 'ttsb.h', Path(__file__)]):
        if f.is_file():
            h.update(f.name.encode())
            h.update(f.read_bytes())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = True) -> Path:
    stamp = OBJ_DIR / 'digest.txt'
    dig = _digest()
    if not force and OUT.exists() and stamp.exists() and stamp.read_text() == dig:
        return OUT
    OBJ_DIR.mkdir(exist_ok=True)
    nvcc = _nvcc()
    srcs = [s for s in SOURCES if (CSRC / s).exists()]

    def compile_one(src: str) -> str:
        obj = OBJ_DIR / (src + '.o')
        cmd = [nvcc, *NVCC_FLAGS, '-I', str(INCLUDE), '-c', str(CSRC / src), '-o', str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f'nvcc failed for {src}:\n{r.stdout}\n{r.stderr}')
        return str(obj)

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [nvcc, '-shared', '-o', str(OUT), *objs, '-gencode', 'arch=compute_90a,code=sm_90a', '-Xcompiler', '-fPIC', '-ldl']
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f'link failed:\n{r.stdout}\n{r.stderr}')
    stamp.write_text(dig)
    if verbose:
        print(f'built {OUT} ({OUT.stat().st_size / 1e6:.1f} MB) from {len(objs)} objects')
    return OUT


if __name__ == '__main__':
    build(force='--force' in sys.argv)
