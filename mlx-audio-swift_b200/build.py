"""In-tree build of libb200audio.so (nvcc, sm_90a only).  No JIT cache, no pip install: the .so
lives next to the sources so it travels with the repo snapshot to the GPU box."""
from __future__ import annotations

import os
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
LIBDIR = HERE / "lib"
LIB = LIBDIR / "libb200audio.so"
SOURCES = ["api.cu", "mel.cu", "snac.cu", "llama.cu", "tc_gemm.cu", "conv_gemm.cu", "whisper.cu", "vocos.cu", "encodec.cu", "weights.cu", "speech_tokenizer.cu", "qwen3_sampler.cu", "speaker_encoder.cu", "mimi.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def _stale(target: Path, deps) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(d).stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    LIBDIR.mkdir(exist_ok=True)
    objdir = HERE / "build"
    objdir.mkdir(exist_ok=True)
    headers = list(CSRC.glob("*.cuh")) + list((HERE.parent / "include").glob("*.h"))
    nvcc = _nvcc()
    objs, procs = [], []
    for src in SOURCES:
        obj = objdir / (src + ".o")
        objs.append(obj)
        if force or _stale(obj, [CSRC / src] + headers):
            cmd = [nvcc, *NVCC_FLAGS, "-c", str(CSRC / src), "-o", str(obj)]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"[b200audio build] {src} failed:\n{out}\n")
        elif verbose or out.strip():
            sys.stderr.write(f"[b200audio build] {src}:\n{out}\n")
    if failed:
        raise RuntimeError("nvcc failed")
    if force or procs or _stale(LIB, objs):
        cmd = [nvcc, "-shared", "-o", str(LIB), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a",
               "-Xcompiler", "-fPIC", "-lcuda"]
        subprocess.run(cmd, check=True)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
