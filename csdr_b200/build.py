"""Builds csdr_b200/libcsdr_b200.so in-tree: nvcc for the kernels + C ABI (sm_90a only), gcc for the
host-side C (filter design, geometry).  The .so is git-ignored: build() makes it."""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
CSRC = PKG / "csrc"
HOST = PKG / "host"
OBJ = PKG / "build"
LIB = PKG / "libcsdr_b200.so"

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--fmad=true", "--expt-relaxed-constexpr", "-diag-suppress", "20281", f"-I{ROOT / 'include'}", f"-I{CSRC}"]
GCC_FLAGS = ["-std=gnu99", "-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC", f"-I{ROOT / 'include'}"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found")


def declared_functions():
    """every function name include/csdr_b200.h declares = the library's export list"""
    import re
    text = (ROOT / "include" / "csdr_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"^\s*#.*$", "", text, flags=re.M)
    names = set()
    for m in re.finditer(r"\b([A-Za-z_][A-Za-z0-9_]*)\s*\(", text):
        if m.group(1) not in {"sizeof", "defined", "if", "while", "for", "return"}:
            names.add(m.group(1))
    return sorted(names)


def _stale(target: Path, deps) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(d).stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    OBJ.mkdir(exist_ok=True)
    headers = list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + list(HOST.glob("*.h")) + [ROOT / "include" / "csdr_b200.h", Path(__file__)]
    objs = []
    for src in sorted(CSRC.glob("*.cu")):
        if src.name.startswith("bench_") or src.name.startswith("tool_"):
            continue
        obj = OBJ / (src.stem + ".o")
        if force or _stale(obj, [src] + headers):
            cmd = [_nvcc()] + NVCC_FLAGS + ["-c", str(src), "-o", str(obj)]
            r = subprocess.run(cmd, capture_output=True, text=True)
            (OBJ / (src.stem + ".ptxas.txt")).write_text(r.stderr)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stderr}")
            if verbose:
                print(r.stderr)
        objs.append(obj)
    for src in sorted(HOST.glob("*.c")):
        if src.name in ("csdr_cli.c", "bankd.c"):                      # programs ON TOP of the C ABI, not part of the library (bankd.c has a main())
            continue
        obj = OBJ / (src.stem + ".host.o")
        if force or _stale(obj, [src] + headers):
            subprocess.run(["gcc"] + GCC_FLAGS + ["-c", str(src), "-o", str(obj)], check=True)
        objs.append(obj)
    if force or _stale(LIB, objs):
        # export exactly what include/csdr_b200.h declares (the drop-in is LD_PRELOADed into other programs: no stray `main`, no mangled internals)
        vs = OBJ / "exports.map"
        vs.write_text("{ global: " + " ".join(n + ";" for n in declared_functions()) + " local: *; };\n")
        stale = OBJ / "bankd.host.o"
        if stale.exists():
            stale.unlink()
        cmd = [_nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-Xlinker", f"--version-script={vs}", "-o", str(LIB)] + [str(o) for o in objs] + ["-lm", "-ldl"]
        subprocess.run(cmd, check=True)
    cli_src = HOST / "csdr_cli.c"
    cli = PKG / "csdr"
    if cli_src.exists() and (force or _stale(cli, [cli_src, LIB] + headers)):
        subprocess.run(["gcc", "-std=gnu99", "-O2", "-Wno-unused-result", f"-I{ROOT / 'include'}", str(cli_src), "-o", str(cli),
                        f"-L{PKG}", "-lcsdr_b200", "-lm", "-Wl,-rpath,$ORIGIN"], check=True)
    bankd_src = HOST / "bankd.c"
    bankd = PKG / "csdr-bankd"
    if bankd_src.exists() and (force or _stale(bankd, [bankd_src, LIB] + headers)):
        subprocess.run(["gcc", "-std=gnu99", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(bankd_src), "-o", str(bankd),
                        f"-L{PKG}", "-lcsdr_b200", "-lm", "-Wl,-rpath,$ORIGIN"], check=True)
    # host/programs/: programs on the C ABI that are not in the host/*.c list every library build compiles (each has a main())
    synth_src = HOST / "programs" / "synth.c"
    synth = PKG / "csdr-synth"
    if synth_src.exists() and (force or _stale(synth, [synth_src, LIB] + headers)):
        subprocess.run(["gcc", "-std=gnu99", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(synth_src), "-o", str(synth),
                        f"-L{PKG}", "-lcsdr_b200", "-lm", "-Wl,-rpath,$ORIGIN"], check=True)
    return LIB


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
