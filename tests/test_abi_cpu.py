"""CPU-side checks of the drop-in boundary: the C-ABI library builds/loads and exports every
symbol that include/adp_b200.h declares, the ctypes argtypes of _lib.SIGNATURES match every prototype,
and the ctypes argument structs match the header's field by field, in names, offsets and sizes (no
compute calls: there is no GPU here)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "adp_b200.h")


def header_text():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def declared_symbols():
    return sorted(set(re.findall(r"\b(adp_[a-z0-9_]+)\s*\(", header_text())))


def structs():
    """header struct name -> its ctypes class"""
    from audio_diffusion_pytorch_b200 import _lib
    return {"adp_conv_gemm_args": _lib.ConvGemmArgs, "adp_stem_in_args": _lib.StemInArgs,
            "adp_stem_out_args": _lib.StemOutArgs, "adp_narrow_conv_args": _lib.NarrowConvArgs,
            "adp_wgrad_args": _lib.WgradArgs, "adp_narrow_conv_bwd_args": _lib.NarrowConvBwdArgs,
            "adp_stem_out_bwd_args": _lib.StemOutBwdArgs, "adp_stem_in_bwd_args": _lib.StemInBwdArgs,
            "adp_attention_bwd_args": _lib.AttentionBwdArgs}


def prototypes():
    """entry point -> list of its parameter declarations, as written in the header"""
    out = {}
    for name, params in re.findall(r"\b(adp_\w+)\s*\(([^)]*)\)\s*;", header_text()):
        params = " ".join(params.split())
        out[name] = [] if params == "void" else [p.strip() for p in params.split(",")]
    return out


def test_header_declares_the_hot_path_entry_points():
    syms = declared_symbols()
    for name in ("adp_conv_gemm", "adp_gn_silu", "adp_ln_film", "adp_attention",
                 "adp_stem_in", "adp_stem_out", "adp_narrow_conv", "adp_sampler_step",
                 "adp_skinny_linear", "adp_time_features"):
        assert name in syms


def test_library_exports_every_declared_symbol():
    from audio_diffusion_pytorch_b200 import _build
    path = _build.build()
    lib = ctypes.CDLL(path)
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, f"declared in include/adp_b200.h but not exported: {missing}"
    lib.adp_version.restype = ctypes.c_int
    assert lib.adp_version() >= 1


def test_ctypes_structs_match_header_field_order():
    text = open(HEADER).read()
    assert sorted(re.findall(r"typedef struct (adp_\w+) \{", text)) == sorted(structs())
    for struct, cls in structs().items():
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), text, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        names = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            for part in decl.split(","):
                names.append(re.sub(r"\[.*\]", "", part.strip().split()[-1].lstrip("*")))
        assert names == [f[0] for f in cls._fields_], (struct, names)


def _argtype(param: str):
    """The ctypes argtype a header parameter declaration calls for."""
    m = re.search(r"\b(adp_\w+_args)\s*\*", param)
    if m:
        return ctypes.POINTER(structs()[m.group(1)])
    if "*" in param or param.split()[0] == "adp_stream_t":
        return ctypes.c_void_p
    kind = " ".join(param.split()[:-1])
    return {"int": ctypes.c_int32, "int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64,
            "float": ctypes.c_float}[kind]


def test_signatures_match_header_prototypes():
    """Every status-returning entry point of the header has a _lib.SIGNATURES entry and every entry a
    prototype, with the same number of arguments, each of the same kind."""
    from audio_diffusion_pytorch_b200 import _lib
    protos = prototypes()
    assert set(protos) == set(declared_symbols())
    assert sorted(_lib.EXPORTS) == sorted(protos)
    assert set(protos) - set(_lib.SIGNATURES) == {"adp_version", "adp_last_error"}
    assert not set(_lib.SIGNATURES) - set(protos), "in _lib.SIGNATURES but not declared"
    wrong = []
    for name, argtypes in _lib.SIGNATURES.items():
        want = [_argtype(p) for p in protos[name]]
        if len(want) != len(argtypes):
            wrong.append(f"{name}: {len(argtypes)} argtypes, {len(want)} parameters")
        wrong += [f"{name} argument {i} ({protos[name][i]}): {g.__name__}, want {w.__name__}"
                  for i, (g, w) in enumerate(zip(argtypes, want)) if g is not w]
    assert not wrong, "\n".join(wrong)


def test_ctypes_struct_layout_matches_c_compiler(tmp_path):
    """sizeof and every field's offsetof, from a C probe compiled against the header, equal ctypes'."""
    cc = next((c for c in (os.environ.get("CC"), "cc", "gcc", "clang") if c and shutil.which(c)), None)
    if cc is None:
        pytest.skip("no C compiler found (CC, cc, gcc, clang) to build the layout probe")
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "adp_b200.h"', "int main(void) {"]
    want = {}
    for struct, cls in structs().items():
        lines.append(f'  printf("{struct} sizeof %zu\\n", sizeof({struct}));')
        want[f"{struct} sizeof"] = ctypes.sizeof(cls)
        for field, _ in cls._fields_:
            lines.append(f'  printf("{struct} {field} %zu\\n", offsetof({struct}, {field}));')
            want[f"{struct} {field}"] = getattr(cls, field).offset
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text("\n".join(lines) + "\n")
    subprocess.run([cc, "-std=c99", "-I", os.path.dirname(HEADER), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    got = {k: int(v) for k, v in (line.rsplit(" ", 1) for line in out.splitlines())}
    assert got.keys() == want.keys()
    wrong = [f"{k}: C {got[k]}, ctypes {want[k]}" for k in want if got[k] != want[k]]
    assert not wrong, "\n".join(wrong)
