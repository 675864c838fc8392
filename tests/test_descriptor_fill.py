"""The launch descriptors of the C ABI: the pointee types of abi.py's mirrors against the headers, and the rules native.fill holds
every descriptor's fields to (dtype of the pointee, NULL only where the header allows it, scalars given, contiguous, one CUDA device)."""
import ctypes as C
import os
import subprocess

import pytest
import torch

import test_host
from vid2player3d_b200 import abi, native

C_NAMES = {C.c_float: "float", C.c_int64: "int64_t", C.c_uint8: "uint8_t", C.c_uint32: "uint32_t", C.c_int32: "int32_t"}
# the descriptors native.fill fills, and a dtype each typed pointer field must refuse
FILLED = ("MotionLibView", "Buffers", "V2PState", "V2PCtrl", "V2PPreStep", "V2PStream", "V2PTaskReset", "V2PActorReset", "V2PRec", "V2PBest",
          "ResetMasked", "MotionState", "MotionContext", "ObsImitation", "ObsRows", "V2PSmpl", "V2PHead", "V2PAero", "V2PBallReset",
          "V2PCtrlReset", "V2PInEst")
DTYPE = {abi.F32P: torch.float32, abi.I64P: torch.int64, abi.U8P: torch.bool, abi.U32P: torch.int32, abi.I32P: torch.int32,
         C.c_void_p: torch.bfloat16}
WRONG = {abi.F32P: torch.float64, abi.I64P: torch.int32, abi.U8P: torch.int32, abi.U32P: torch.int64, abi.I32P: torch.int64}


def fields(kind):
    """(struct, field) of every descriptor native.fill fills: its pointer fields, typed pointer fields or scalar fields without a default"""
    out = []
    for name in FILLED:
        S = getattr(abi, name)
        for f, ct in S._fields_:
            ptr = issubclass(ct, C.c_void_p)
            if {"ptr": ptr, "typed": ptr and ct is not C.c_void_p, "scalar": not ptr and f not in S._defaults_}[kind]:
                out.append(pytest.param(name, f, id=f"{name}.{f}"))
    return out


def valid(name, device="cpu"):
    """(S, scalars, tensors) that fill accepts on a CUDA device: every field but the defaulted scalars, a tensor of its pointee's dtype
    for every pointer"""
    S = getattr(abi, name)
    scalars, tensors = {}, {}
    for f, ct in S._fields_:
        if issubclass(ct, C.c_void_p):
            tensors[f] = torch.zeros(4, dtype=DTYPE[ct], device=device)
        elif f not in S._defaults_:
            scalars[f] = [2] * ct._length_ if issubclass(ct, C.Array) else 3
    return S, scalars, tensors


def pointee_mismatches(tmp_path):
    """the pointer fields of abi.py's mirrors whose pointee class is not the headers' pointee type (gcc's __builtin_types_compatible_p
    on *((T*)0)->f, which ignores const); an untyped c_void_p field must be void* / const void* or point at a mirrored struct"""
    mirrors = [(getattr(abi, cls), ctype) for mod, cls, ctype in test_host.STRUCT_MIRRORS if mod == "abi"]
    structs = [ctype for _, ctype in mirrors]
    lines, want = [], []
    for S, ctype in mirrors:
        for f, ct in S._fields_:
            if not issubclass(ct, C.c_void_p):
                continue
            p = f"(({ctype}*)0)->{f}"
            tests = [(f"__builtin_types_compatible_p(__typeof__(*{p}), {c})", c) for c in C_NAMES.values()]
            tests += [(f"__builtin_types_compatible_p(__typeof__({p}), {q}{t}*)", "void" if t == "void" else "struct")
                      for t in ("void",) + tuple(structs) for q in ("", "const ")]
            expr = " : ".join(f'{e} ? "{n}"' for e, n in tests) + ' : "other"'
            lines.append(f'printf("%s\\n", {expr});')
            want.append((f"{ctype}.{f}", ct))
    src, exe = tmp_path / "pointee.c", tmp_path / "pointee"
    src.write_text("#include <stdio.h>\n" + "".join(f'#include "{h}"\n' for h in test_host.ENV_HEADERS) + "int main(void) {\n" +
                   "\n".join(lines) + "\nreturn 0;\n}\n")
    subprocess.check_call(["gcc", "-w", "-I", os.path.join(test_host.ROOT, "include"), str(src), "-o", str(exe)])
    got = subprocess.check_output([str(exe)], text=True).splitlines()
    assert len(got) == len(want)
    return [f"{field}: mirror {ct.__name__}, header {g}" for (field, ct), g in zip(want, got)
            if g not in (("void", "struct") if ct is C.c_void_p else (C_NAMES[ct.pointee],))]


def test_pointer_fields_carry_the_headers_pointee_types(tmp_path):
    assert pointee_mismatches(tmp_path) == []


def test_pointee_check_rejects_a_retyped_field(tmp_path, monkeypatch):
    """negative control: a mirror of b200v2p_state_t with root_pos (float*) declared int64_t*"""
    f = [(n, abi.I64P if n == "root_pos" else ct) for n, ct in abi.V2PState._fields_]
    assert dict(abi.V2PState._fields_)["root_pos"] is abi.F32P
    monkeypatch.setattr(abi, "V2PState", type("V2PState", (C.Structure,), {"_fields_": f}))
    assert pointee_mismatches(tmp_path) == ["b200v2p_state_t.root_pos: mirror I64P, header float"]


@pytest.mark.parametrize("name", FILLED)
def test_nullable_and_default_names_are_fields(name):
    S = getattr(abi, name)
    kind = {f: issubclass(ct, C.c_void_p) for f, ct in S._fields_}
    assert all(kind.get(f) is True for f in S._nullable_) and all(kind.get(f) is False for f in S._defaults_)


@pytest.mark.parametrize("name,field", fields("typed"))
def test_fill_refuses_a_wrong_dtype(name, field):
    S, scalars, tensors = valid(name)
    tensors[field] = torch.zeros(4, dtype=WRONG[dict(S._fields_)[field]])
    with pytest.raises(ValueError, match=rf"^{name}\.{field}: torch\.\w+, the header's pointee needs"):
        native.fill(S, scalars, tensors)


@pytest.mark.parametrize("name,field", fields("ptr"))
def test_fill_refuses_none_where_the_header_allows_no_null(name, field):
    S, scalars, tensors = valid(name)
    tensors[field] = None
    want = r"not on the CUDA device" if field in S._nullable_ else rf"^{name}\.{field}: None"
    with pytest.raises(ValueError, match=want):
        native.fill(S, scalars, tensors)
    del tensors[field]                                      # a missing key is None
    with pytest.raises(ValueError, match=want):
        native.fill(S, scalars, tensors)


@pytest.mark.parametrize("name,field", fields("scalar"))
def test_fill_refuses_a_missing_scalar(name, field):
    S, scalars, tensors = valid(name)
    del scalars[field]
    with pytest.raises(ValueError, match=rf"^{name}\.{field}: missing"):
        native.fill(S, scalars, tensors)


@pytest.mark.parametrize("name,field", fields("ptr"))
def test_fill_refuses_a_non_contiguous_tensor(name, field):
    S, scalars, tensors = valid(name)
    tensors[field] = torch.zeros(4, 2, dtype=tensors[field].dtype)[:, 0]
    with pytest.raises(ValueError, match=rf"^{name}\.{field}: not contiguous"):
        native.fill(S, scalars, tensors)


@pytest.mark.parametrize("name", FILLED)
def test_fill_refuses_valid_cpu_tensors_for_the_device_only(name):
    S, scalars, tensors = valid(name)
    first = next(f for f, ct in S._fields_ if issubclass(ct, C.c_void_p))
    with pytest.raises(ValueError, match=rf"^{name}\.{first}: not on the CUDA device"):
        native.fill(S, scalars, tensors)


@pytest.mark.gpu
@pytest.mark.parametrize("name", FILLED)
def test_fill_writes_every_field(name):
    """on the device: every pointer is its tensor's address (NULL for a None), every scalar its value, the defaulted ones 0; a tensor
    on the host among them is refused"""
    S, scalars, tensors = valid(name, "cuda:0")
    null = S._nullable_[:1]
    s = native.fill(S, scalars, {f: None if f in null else t for f, t in tensors.items()})
    for f, ct in S._fields_:
        got = getattr(s, f)
        if issubclass(ct, C.c_void_p):
            assert (got if ct is C.c_void_p else got.value) == (None if f in null else tensors[f].data_ptr()), f
        elif f in S._defaults_:
            assert (list(got) == [0] * ct._length_) if issubclass(ct, C.Array) else got == 0, f
        else:
            assert (list(got) == scalars[f]) if issubclass(ct, C.Array) else got == scalars[f], f
    last = [f for f, ct in S._fields_ if issubclass(ct, C.c_void_p)][-1]
    with pytest.raises(ValueError, match=rf"^{name}\.{last}: not on the CUDA device"):
        native.fill(S, scalars, dict(tensors, **{last: tensors[last].cpu()}))
