"""Build a host library that EXECUTES the shipped .cu files under tests/host_shim/cuda_emul.h (CPU test tier; test infrastructure only).

The kernel sources are used as they are; only two CUDA-only spellings are rewritten on the fly, textually:
    kernel<<<grid, block, smem, stream>>>(args)   ->   ::cuda_emul::cfg(grid, block, smem, stream).run(kernel, args)
    extern __shared__ __align__(N) unsigned char name[];   ->   unsigned char* name = ::cuda_emul::dyn_smem();
so the launchers (grid and shared-memory arithmetic, dispatch on sizes) run too.  The wrappers appended after the sources export plain C
entry points for ctypes.
"""
import re
import shutil
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent.parent
CSRC = ROOT / "csdr_b200" / "csrc"
SHIM = ROOT / "tests" / "host_shim"
CUDA_INC = Path("/usr/local/cuda/include")

_LAUNCH = re.compile(r"([A-Za-z_][\w:]*(?:<[^<>;(){}]*>)?)\s*<<<(.+?)>>>\s*\(", re.S)
_DYN = re.compile(r"extern\s+__shared__\s+(?:__align__\(\d+\)\s+)?unsigned\s+char\s+(\w+)\[\];")


def transform(text: str) -> str:
    text = _DYN.sub(lambda m: f"unsigned char* {m.group(1)} = ::cuda_emul::dyn_smem();", text)
    return _LAUNCH.sub(lambda m: f"::cuda_emul::cfg({m.group(2)}).run({m.group(1)}, ", text)


import os

# CUDA_EMUL_SANITIZE=1: build the emulated code with UBSan (misaligned float4/float2 accesses, out-of-range shifts, signed overflow ...) and
# abort on the first report -- alignment is what a CPU would otherwise forgive and a GPU would not
SANITIZE = ["-fsanitize=undefined", "-fno-sanitize-recover=all", "-fno-sanitize=vptr"] if os.environ.get("CUDA_EMUL_SANITIZE") else []


def available() -> bool:
    return bool(shutil.which("g++")) and (CUDA_INC / "cuda_runtime.h").exists()


PRELUDE = """#include <algorithm>
#include <cstdarg>
using std::max;
using std::min;
#include "cuda_emul.h"
#include "../../csdr_b200/csrc/common.cuh"
namespace csdrb {
static char g_emul_error[512];
void set_error(const char* fmt, ...) { va_list ap; va_start(ap, fmt); vsnprintf(g_emul_error, sizeof g_emul_error, fmt, ap); va_end(ap); }
int cuda_fail(cudaError_t, const char* what, const char*, int) { set_error("cuda_emul: %s failed", what); return -100; }
}
extern "C" const char* emul_last_error(void) { return csdrb::g_emul_error; }
extern "C" int cuda_emul_take_launch_error(void) { return cuda_emul::take_launch_error() ? 1 : 0; }
extern "C" long emul_barriers(void) { return cuda_emul::st().barriers; }
"""


def build(out_dir: Path, name: str, cu_files, wrappers: str, extra_includes=(), host_c=()) -> Path:
    """one translation unit: prelude, the transformed .cu files, the extern "C" wrappers"""
    parts = [PRELUDE]
    for inc in extra_includes:
        parts.append(f'#include "{inc}"\n')
    for cu in cu_files:
        src = transform((CSRC / cu).read_text())
        src = src.replace('#include "', f'#include "{CSRC}/')                     # the sources include their neighbours by bare name
        parts.append(f"// ======== {cu} (transformed) ========\n{src}\n")
    parts.append(wrappers)
    cpp = out_dir / f"{name}.cpp"
    cpp.write_text("\n".join(parts))
    so = out_dir / f"{name}.so"
    objs = []
    for c in host_c:                                                               # host C of the product that a launcher calls (filter tables ...)
        obj = out_dir / (Path(c).stem + ".o")
        subprocess.run(["gcc", "-std=gnu99", "-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC", f"-I{ROOT / 'include'}", "-c", str(ROOT / c), "-o", str(obj)],
                       check=True, capture_output=True)
        objs.append(str(obj))
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w"] + SANITIZE + [f"-I{CUDA_INC}", f"-I{SHIM}", f"-I{CSRC}",
                        f"-I{ROOT / 'include'}", str(cpp), str(SHIM / "cuda_emul_runtime.cpp")] + objs + ["-o", str(so), "-lm", "-Wl,-Bsymbolic"], capture_output=True, text=True)   # -Bsymbolic: our cuda* stubs, not a libcudart another test loaded
    if r.returncode != 0:
        raise RuntimeError(f"g++ failed for {name}:\n{r.stderr[-4000:]}")
    return so


# ---- wrappers generated from the launcher prototypes of csdr_b200/csrc/kernels.h ----------------------------------------------------
_PROTO = re.compile(r"^(int|size_t|void)\s+(\w+)\s*\(([^;{}]*?)\)\s*;", re.S | re.M)


def launcher_prototypes():
    text = (CSRC / "kernels.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"//[^\n]*", "", text)
    protos = {}
    for ret, name, args in _PROTO.findall(text):
        params = []
        for a in [x.strip() for x in args.replace("\n", " ").split(",") if x.strip()]:
            m = re.match(r"(.*?)(\w+)$", a)
            params.append((m.group(1).strip(), m.group(2)))
        protos[name] = (ret, params)
    return protos


def _ctype(ctype_text: str):
    import ctypes as C
    t = ctype_text.replace("const", "").strip()
    if "*" in t or t == "cudaStream_t":
        return C.c_void_p
    return {"int": C.c_int, "long": C.c_long, "float": C.c_float, "size_t": C.c_size_t, "bool": C.c_bool}[t]


def build_file(out_dir: Path, cu: str, extra: str = "", host_c=()):
    """library for one .cu file: every launcher of kernels.h that the file defines is exported as emul_<name> (stream argument dropped)"""
    import ctypes as C
    text = (CSRC / cu).read_text()
    protos = {n: p for n, p in launcher_prototypes().items() if re.search(r"\b%s\s*\(" % n, text) and re.search(r"^\w[\w\s\*]*\b%s\s*\(" % n, text, re.M)}
    w = []
    for name, (ret, params) in protos.items():
        decl = ", ".join(f"{t} {n}" for t, n in params if t != "cudaStream_t")
        call = ", ".join("nullptr" if t == "cudaStream_t" else n for t, n in params)
        body = f"csdrb::{name}({call});" if ret == "void" else f"return csdrb::{name}({call});"
        w.append(f'extern "C" {ret} emul_{name}({decl}) {{ {body} }}')
    so = build(out_dir, "emul_" + Path(cu).stem, [cu], "\n".join(w) + "\n" + extra, host_c=host_c)
    lib = C.CDLL(str(so))
    for name, (ret, params) in protos.items():
        f = getattr(lib, "emul_" + name)
        f.argtypes = [_ctype(t) for t, n in params if t != "cudaStream_t"]
        f.restype = {"int": C.c_int, "size_t": C.c_size_t, "void": None}[ret]
    lib.emul_last_error.restype = C.c_char_p
    lib.emul_barriers.restype = C.c_long
    return lib, sorted(protos)


# ---- the whole library under emulation: libcsdr_b200_emul.so with the real C ABI, plus the CLI linked against it ----------------------
PRELUDE_FULL = """#include <algorithm>
using std::max;
using std::min;
#include "cuda_emul.h"
"""


def build_full(out_dir: Path):
    """Every product translation unit (kernels, launchers, csrc/capi.cu, host C) compiled for the host under cuda_emul.h and linked into
    ONE shared library that exports the product's C ABI, so host-side code on top of the ABI (the csdr CLI, Part A's workspace in dropin.cu,
    the streaming logic in capi.cu) runs in the CPU tier.  Returns (library path, CLI path).  Test artefacts only -- built into a temporary
    directory, never installed next to the product."""
    from concurrent.futures import ThreadPoolExecutor
    out_dir.mkdir(exist_ok=True)
    cus = sorted(p.name for p in CSRC.glob("*.cu") if not p.name.startswith(("bench_", "tool_")))

    def compile_cu(cu):
        src = transform((CSRC / cu).read_text()).replace('#include "', f'#include "{CSRC}/')
        src = src.replace(f'#include "{CSRC}/csdr_b200.h"', '#include "csdr_b200.h"')
        cpp = out_dir / f"full_{Path(cu).stem}.cpp"
        hook = 'extern "C" int cuda_emul_take_launch_error(void) { return cuda_emul::take_launch_error() ? 1 : 0; }\n' if cu == "capi.cu" else ""
        cpp.write_text(PRELUDE_FULL + hook + src)
        obj = cpp.with_suffix(".o")
        r = subprocess.run(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-w"] + SANITIZE + [f"-I{CUDA_INC}", f"-I{SHIM}", f"-I{CSRC}",
                            f"-I{ROOT / 'include'}", "-c", str(cpp), "-o", str(obj)], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"g++ failed for {cu}:\n{r.stderr[-3000:]}")
        return str(obj)

    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(compile_cu, cus))
    rt = out_dir / "cuda_emul_runtime.o"
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-w", f"-I{CUDA_INC}", "-c", str(SHIM / "cuda_emul_runtime.cpp"), "-o", str(rt)], check=True, capture_output=True)
    host = []
    for c in sorted((ROOT / "csdr_b200" / "host").glob("*.c")):
        if c.name in ("csdr_cli.c", "bankd.c"):
            continue
        obj = out_dir / (c.stem + ".host.o")
        subprocess.run(["gcc", "-std=gnu99", "-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC", f"-I{ROOT / 'include'}", "-c", str(c), "-o", str(obj)],
                       check=True, capture_output=True)
        host.append(str(obj))
    lib = out_dir / "libcsdr_b200_emul.so"
    r = subprocess.run(["g++", "-shared"] + SANITIZE + ["-o", str(lib)] + objs + [str(rt)] + host + ["-lm", "-lpthread", "-ldl", "-Wl,-Bsymbolic"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stderr[-3000:])
    cli = out_dir / "csdr_emul"
    subprocess.run(["gcc", "-std=gnu99", "-O2", "-Wno-unused-result", f"-I{ROOT / 'include'}", str(ROOT / "csdr_b200" / "host" / "csdr_cli.c"), "-o", str(cli),
                    f"-L{out_dir}", "-lcsdr_b200_emul", "-lm", f"-Wl,-rpath,{out_dir}"], check=True, capture_output=True)
    bankd_src = ROOT / "csdr_b200" / "host" / "bankd.c"
    if bankd_src.exists():                                                 # the ingest daemon is plain C on the ABI too
        subprocess.run(["gcc", "-std=gnu99", "-O2", "-Wall", f"-I{ROOT / 'include'}", str(bankd_src), "-o", str(out_dir / "csdr-bankd_emul"),
                        f"-L{out_dir}", "-lcsdr_b200_emul", "-lm", f"-Wl,-rpath,{out_dir}"], check=True, capture_output=True)
    return lib, cli


_full = None


def build_full_once(tmp_path_factory):
    """one build of the whole emulated library per test process, shared by the modules that need it"""
    global _full
    if _full is None:
        _full = build_full(tmp_path_factory.mktemp("emul_full"))
    return _full


_ABSENT = object()


def _swap(obj, key, value):
    """set obj.key (a module) or obj[key] (a list or dict) to value, or delete it for _ABSENT; returns what was there"""
    if isinstance(obj, (list, dict)):
        old = obj[key] if isinstance(obj, list) or key in obj else _ABSENT
        if value is _ABSENT:
            del obj[key]
        else:
            obj[key] = value
    else:
        old = getattr(obj, key, _ABSENT)
        if value is _ABSENT:
            delattr(obj, key)
        else:
            setattr(obj, key, value)
    return old


def emulated_bankd(tmp_path_factory, patches=lambda lib, cli: ()):
    """Generator behind the module fixtures of tests/test_bankd_*_emulated.py: csdr-bankd linked against the emulated library, with two pretend
    devices for --devices (CUDA_EMUL_DEVICES=2) and a memcpy stand-in for NCCL (fake_nccl.c), both inherited by the daemon.  patches(lib, cli)
    lists (module or container, name or key, value) to set while the module's tests run, e.g. its MULTI_DEVICES.  Yields the daemon's path;
    afterwards every patched attribute is restored and the environment variables are cleared."""
    import os
    import pytest
    if not available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, cli = build_full_once(tmp_path_factory)
    fake = tmp_path_factory.mktemp("fake_nccl") / "libfake_nccl.so"
    subprocess.run(["gcc", "-O1", "-fPIC", "-shared", str(SHIM / "fake_nccl.c"), "-o", str(fake)], check=True)
    saved = [(obj, key, _swap(obj, key, value)) for obj, key, value in patches(lib, cli)]
    os.environ["CUDA_EMUL_DEVICES"] = "2"
    os.environ["CSDRB_NCCL_LIB"] = str(fake)
    try:
        yield str(lib.parent / "csdr-bankd_emul")
    finally:
        for obj, key, old in reversed(saved):
            _swap(obj, key, old)
        del os.environ["CUDA_EMUL_DEVICES"], os.environ["CSDRB_NCCL_LIB"]
