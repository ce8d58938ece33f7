"""CPU test: the C-ABI library builds (nvcc cross-compiles sm_90a without a GPU), loads, and exports every function
include/musev_b200.h declares. No compute call is made."""
import ctypes
import os
import re
import subprocess

from conftest import ROOT


def _declared_functions():
    src = open(os.path.join(ROOT, "include", "musev_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = re.findall(r"\b(mvb_[a-z0-9_]+)\s*\(", src)
    return sorted(set(n for n in names))


def test_header_declares_expected_surface():
    names = _declared_functions()
    for must in ("mvb_create", "mvb_load_weight", "mvb_finalize", "mvb_workspace_bytes", "mvb_unet_forward",
                 "mvb_fuse_cfg_ddim", "mvb_destroy", "mvb_last_error", "mvb_op_conv_gemm", "mvb_op_attention", "mvb_debug_attention_trace", "mvb_tensor_map_cache_stats",
                 "mvb_op_groupnorm", "mvb_op_groupnorm_fused", "mvb_op_layernorm", "mvb_op_softmax_rows"):
        assert must in names


def test_library_loads_and_exports_every_symbol(built_lib):
    lib = ctypes.CDLL(built_lib)
    for name in _declared_functions():
        assert hasattr(lib, name), f"{name} declared in include/musev_b200.h but not exported"
    lib.mvb_version.restype = ctypes.c_int
    assert lib.mvb_version() >= 1


def test_library_is_native_sm90a(built_lib):
    sass = subprocess.run(["cuobjdump", "-sass", built_lib], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    for mnemonic in ("HGMMA", "UTMALDG", "SYNCS"):           # wgmma / TMA / mbarrier
        assert mnemonic in sass, mnemonic


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "musev_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "from oracle" not in txt and "import oracle" not in txt, f


def test_struct_layouts_match_ctypes_mirrors(tmp_path):
    """Every struct of include/musev_b200.h against its ctypes mirror: size and the offset of every field, as a C compiler sees
    them (gcc on the header alone -- the boundary is plain C). Guards the Python binding against silent ABI drift."""
    from musev_b200 import _capi
    mirrors = {"mvb_conv_gemm_desc": _capi.ConvGemmDesc, "mvb_attention_desc": _capi.AttentionDesc, "mvb_config": _capi.MvbConfig,
               "mvb_unet_args": _capi.MvbUnetArgs, "mvb_named_tensor": _capi.MvbNamedTensor,
               "mvb_controlnet_args": _capi.MvbControlnetArgs, "mvb_vae_decode_args": _capi.MvbVaeDecodeArgs}
    header = open(os.path.join(ROOT, "include", "musev_b200.h")).read()
    declared = set(re.findall(r"^\}\s*(mvb_[a-z_]+);", header, flags=re.M))
    assert declared == set(mirrors), declared ^ set(mirrors)
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "musev_b200.h"', "int main(void) {"]
    for cname, cls in mirrors.items():
        lines.append(f'  printf("{cname} . %zu\\n", sizeof({cname}));')
        for fname, *_ in cls._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    r = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    for line in out.strip().splitlines():
        cname, fname, value = line.split()
        cls = mirrors[cname]
        expect = ctypes.sizeof(cls) if fname == "." else getattr(cls, fname).offset
        assert int(value) == expect, (cname, fname, int(value), expect)


def _prototypes():
    """name -> number of parameters, parsed from the header (comments stripped; `void` = 0)."""
    src = open(os.path.join(ROOT, "include", "musev_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(mvb_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", src):
        args = m.group(2).strip()
        protos[m.group(1)] = 0 if args in ("", "void") else args.count(",") + 1
    return protos


def test_ctypes_argtypes_match_header_prototypes(built_lib):
    """Every binding the Python host side declares has as many `argtypes` as the C prototype has parameters."""
    from musev_b200 import _capi
    lib = _capi.lib()
    protos = _prototypes()
    bound = 0
    for name, nparams in protos.items():
        fn = getattr(lib, name)
        if fn.argtypes is None:
            continue                      # C-only entry (not called from the Python mirror)
        bound += 1
        assert len(fn.argtypes) == nparams, (name, len(fn.argtypes), nparams)
    assert bound >= 25, bound
