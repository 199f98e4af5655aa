"""include/cook_gpu.h against its ctypes mirror, cook_b200/abi.py (CPU only; the C compiler reads the header).

Prototypes: every int32_t entry point of the header has abi.ARGTYPES, and each parameter's C spelling maps to its
ctypes type through one table.  Layouts: every ctypes Structure of abi.py is paired with its typedef; its size and
each field's offset, size, pointee size and type are compared with one compiled C unit.  Constants: every value abi.py
mirrors from the header.  Exports: libcookgpu.so binds every entry point with these types (when it is built).
"""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from cook_b200 import abi, engine
from cook_b200.engine import GpuEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "cook_gpu.h")

# every ctypes Structure of abi.py and the typedef it mirrors
STRUCTS = {abi.GpuConfig: "cook_gpu_config", abi.TasksSoA: "cook_tasks_soa", abi.UserTable: "cook_user_table",
           abi.PoolQuota: "cook_pool_quota", abi.RankParams: "cook_rank_params", abi.JobsSoA: "cook_jobs_soa",
           abi.OffersSoA: "cook_offers_soa", abi.Groups: "cook_groups", abi.MatchParams: "cook_match_params",
           abi.MatchStats: "cook_match_stats", abi.FailureCounts: "cook_failure_counts",
           abi.RunningSoA: "cook_running_soa", abi.HostTable: "cook_host_table",
           abi.RebalanceParams: "cook_rebalance_params", abi.Decision: "cook_decision", abi.RebTrace: "cook_reb_trace",
           abi.StateDelta: "cook_state_delta", abi.ConsiderableParams: "cook_considerable_params", abi.Fp: "cook_fp",
           abi.StateDigest: "cook_state_digest_out", abi.JobsRows: "cook_jobs_rows", abi.TasksRows: "cook_tasks_rows",
           abi.StateRows: "cook_state_rows", abi.StateSizes: "cook_state_sizes", abi.PhaseStats: "cook_phase_stats"}

# the header's C spelling of a type (without const and *) -> ctypes; None: an opaque handle or void (c_void_p)
BASE = {"int32_t": C.c_int32, "int64_t": C.c_int64, "uint8_t": C.c_uint8, "uint64_t": C.c_uint64,
        "double": C.c_double, "char": C.c_char, "void": None, "cook_ctx": None, "cook_pool": None,
        **{c: s for s, c in STRUCTS.items()}}
C_OF = {t: c for c, t in BASE.items() if t is not None}


def ctype_of(spelling):
    """'const cook_user_table*' -> POINTER(abi.UserTable); 'cook_pool*', 'void*' -> c_void_p; 'char*' -> c_char_p."""
    s = spelling.replace("const", " ").replace(" ", "")
    base = s.rstrip("*")
    t, stars = BASE[base], len(s) - len(base)
    if t is None or t is C.c_char:
        t, stars = C.c_void_p if t is None else C.c_char_p, stars - 1
    for _ in range(stars):
        t = C.POINTER(t)
    return t


def _header():
    return re.sub(r"/\*.*?\*/", " ", open(HDR).read(), flags=re.S)


def prototypes():
    """{entry point: [(C type, parameter name)]} of every int32_t function the header declares."""
    out = {}
    for name, args in re.findall(r"int32_t\s+(cook_\w+)\s*\(([^)]*)\)\s*;", _header()):
        params = []
        for p in args.split(","):
            m = re.fullmatch(r"(.*?)\s*(\w+)\s*(\[\d+\])?", " ".join(p.split()))
            params.append((m.group(1) + ("*" if m.group(3) else ""), m.group(2)))
        out[name] = params
    return out


def header_constants():
    return re.findall(r"\b(COOK_[A-Z0-9_]+)\s*=", _header())


def abi_name(const):
    """The abi.py name of a header constant: COOK_OK and COOK_E_* keep theirs, the others drop COOK_."""
    return const if const == "COOK_OK" or const.startswith("COOK_E_") else const[len("COOK_"):]


# ---- prototypes ------------------------------------------------------------------------------------------------
def test_every_entry_point_has_bindings():
    assert sorted(prototypes()) == sorted(abi.ARGTYPES)


@pytest.mark.parametrize("name", sorted(abi.ARGTYPES))
def test_prototype(name):
    assert [ctype_of(t) for t, _ in prototypes()[name]] == abi.ARGTYPES[name]


def test_derived_prototypes_are_the_plain_ones():
    protos = prototypes()
    for plain in ("cook_state_match", "cook_state_rebalance"):
        assert protos[plain + "_derived"] == protos[plain]           # the same arguments, names included
    assert "derived" in GpuEngine.state_match.__code__.co_varnames
    assert "derived" in GpuEngine.state_rebalance.__code__.co_varnames


# ---- one compiled unit: layouts, derived prototypes, constants ---------------------------------------------------
def _field_lines(cls, cname):
    """printf lines of (key, value): sizeof, each field's offset, size, pointee size and type compatibility."""
    out = [(f"{cname}", f"sizeof({cname})")]
    for f, t in cls._fields_:
        x = f"(({cname}*)0)->{f}"
        out += [(f"{cname}.{f}.offset", f"offsetof({cname}, {f})"), (f"{cname}.{f}.size", f"sizeof({x})")]
        if issubclass(t, C._Pointer):
            out += [(f"{cname}.{f}.pointee", f"sizeof(*{x})"), (f"{cname}.{f}.type", (f"*{x}", t._type_))]
        elif issubclass(t, C.Array):
            out.append((f"{cname}.{f}.type", (f"{x}[0]", t._type_)))
        else:
            out.append((f"{cname}.{f}.type", (x, t)))
    return [(k, v if isinstance(v, str) else
             f"__builtin_types_compatible_p(__typeof__({v[0]}), {C_OF[v[1]]})") for k, v in out]


def _want(cls, cname):
    want = {cname: C.sizeof(cls)}
    for f, t in cls._fields_:
        d = getattr(cls, f)
        want.update({f"{cname}.{f}.offset": d.offset, f"{cname}.{f}.size": d.size, f"{cname}.{f}.type": 1})
        if issubclass(t, C._Pointer):
            want[f"{cname}.{f}.pointee"] = C.sizeof(t._type_)
    return want


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """Every key of _field_lines and every header constant, as the C compiler evaluates them."""
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    lines = [kv for cls, cname in STRUCTS.items() for kv in _field_lines(cls, cname)]
    lines += [(k, f"(long long){k}") for k in header_constants()]
    lines += [(f"{p}_derived", f"__builtin_types_compatible_p(__typeof__({p}), __typeof__({p}_derived))")
              for p in ("cook_state_match", "cook_state_rebalance")]
    d = tmp_path_factory.mktemp("abi")
    (d / "abi.c").write_text('#include <stddef.h>\n#include <stdio.h>\n#include "cook_gpu.h"\nint main(void) {\n' +
                             "".join(f'  printf("{k} %lld\\n", (long long)({v}));\n' for k, v in lines) +
                             "  return 0;\n}\n")
    subprocess.check_call([cc, "-std=gnu11", "-I", os.path.join(ROOT, "include"), str(d / "abi.c"), "-o", str(d / "abi")])
    return {k: int(v) for k, v in (x.split() for x in subprocess.check_output([str(d / "abi")]).decode().splitlines())}


def test_every_structure_is_paired():
    structs = {v for v in vars(abi).values()
               if isinstance(v, type) and issubclass(v, C.Structure) and v is not abi._SoA}
    assert structs == set(STRUCTS)


@pytest.mark.parametrize("cls", list(STRUCTS), ids=lambda c: c.__name__)
def test_struct_layout(cls, compiled):
    want = _want(cls, STRUCTS[cls])
    assert {k: compiled[k] for k in want} == want


def test_struct_facts():
    assert [n for n, _ in abi.StateDelta._fields_][-2:] == ["running_group_off", "running_group_idx"]
    assert abi.JobsRows._fields_ == abi.JobsSoA._fields_[1:] and abi.TasksRows._fields_ == abi.TasksSoA._fields_[1:]
    assert C.sizeof(abi.Fp) == abi.FP_DTYPE.itemsize == 24


def test_derived_prototypes_compile_as_the_plain_ones(compiled):
    assert compiled["cook_state_match_derived"] == compiled["cook_state_rebalance_derived"] == 1


def test_constants(compiled):
    consts = header_constants()
    mirrored = {abi_name(k): k for k in consts if hasattr(abi, abi_name(k))}
    assert {n: getattr(abi, n) for n in mirrored} == {n: compiled[k] for n, k in mirrored.items()}
    # every constant abi.py states (but INT64_MAX) is the header's
    own = {n for n, v in vars(abi).items() if n.isupper() and isinstance(v, int) and n != "INT64_MAX"}
    assert own <= set(mirrored)
    assert {"PHASE_AUDIT", "AUDIT_N", "USAGE_LAST_MATCH", "FAILC_N", "COOK_E_TOO_LARGE"} <= set(mirrored)
    # abi.AUDIT_NAMES is indexed by COOK_AUDIT_*; ENTRIES and FLAGS start a run of names
    runs = {"ENTRIES": "entries_", "FLAGS": "flag_"}
    for k in consts:
        stem = k[len("COOK_AUDIT_"):]
        if k.startswith("COOK_AUDIT_") and stem != "N":
            name = abi.AUDIT_NAMES[compiled[k]]
            assert name.startswith(runs[stem]) if stem in runs else name == stem.lower(), k
    assert abi.PHASE_CONSIDERABLE == abi.PHASE_COTASKS + 1


# ---- exports ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(engine.LIB_PATH):
        pytest.skip("libcookgpu.so not built")
    return engine.load_library()


@pytest.mark.parametrize("name", sorted(abi.ARGTYPES))
def test_exported(name, lib):
    fn = getattr(lib, name)
    assert fn.restype is C.c_int32 and list(fn.argtypes) == abi.ARGTYPES[name]


def test_version_and_methods(lib):
    assert lib.cook_gpu_version.restype is C.c_char_p and b"sm_90a" in lib.cook_gpu_version()
    for m in ("state_apply", "state_launch", "state_patch", "state_rank", "state_match", "state_rebalance",
              "state_usage", "state_cotasks", "state_considerable", "state_digest", "state_export", "state_queue"):
        assert callable(getattr(GpuEngine, m)), m
