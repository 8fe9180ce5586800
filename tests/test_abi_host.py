"""The ctypes mirror of the C ABI (particles_b200/_lib.py) against include/smcb.h, in one place: every descriptor's
layout as the C compiler lays it out, the kinds of every prototype's return value and arguments, every integer
#define, and the symbols the built library exports.  A wrong mirror does not fail loudly at run time (a field at the
wrong offset or an int bound as int64_t reaches the device as bad memory), so it fails here.  The comparisons are plain
functions that return what disagrees; the last tests feed each a deliberately broken mirror and check that it reports
the break."""
import ctypes as C
import os
import re
import subprocess

import pytest

from particles_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "include", "smcb.h")) as f:
    HEADER = f.read()

# every `typedef struct { ... } smcb_*;` of the header and the ctypes class that mirrors it
STRUCTS = {
    "smcb_vs_desc": _lib.VsDesc,
    "smcb_filter_desc": _lib.FilterDesc,
    "smcb_smooth_desc": _lib.SmoothDesc,
    "smcb_online_desc": _lib.OnlineDesc,
    "smcb_twofilter_desc": _lib.TwoFilterDesc,
    "smcb_variance_desc": _lib.VarDesc,
    "smcb_batch_desc": _lib.BatchDesc,
    "smcb_bank_desc": _lib.BankDesc,
    "smcb_csmc_desc": _lib.CsmcDesc,
    "smcb_hmm_desc": _lib.HmmDesc,
    "smcb_kalman_desc": _lib.KalmanDesc,
}

# every integer `#define SMCB_*` of the header and its Python value
CONSTANTS = {
    "SMCB_OK": _lib.OK, "SMCB_EINVAL": _lib.EINVAL, "SMCB_ECUDA": _lib.ECUDA, "SMCB_ENOSYS": _lib.ENOSYS,
    "SMCB_LSE_SUM": _lib.LSE_SUM, "SMCB_LSE_MEAN": _lib.LSE_MEAN, "SMCB_LSE_ESSL": _lib.LSE_ESSL,
    "SMCB_RS_MULTINOMIAL": _lib.RS_CODES["multinomial"], "SMCB_RS_STRATIFIED": _lib.RS_CODES["stratified"],
    "SMCB_RS_SYSTEMATIC": _lib.RS_CODES["systematic"], "SMCB_RS_RESIDUAL": _lib.RS_CODES["residual"],
    "SMCB_RS_SSP": _lib.RS_CODES["ssp"],
    "SMCB_FK_BOOTSTRAP": _lib.FK_BOOTSTRAP, "SMCB_FK_GUIDED": _lib.FK_GUIDED, "SMCB_FK_APF": _lib.FK_APF,
    "SMCB_FK_AUXBOOT": _lib.FK_AUXBOOT,
    "SMCB_MODEL_STOCHVOL": _lib.MODEL_STOCHVOL, "SMCB_MODEL_LINGAUSS": _lib.MODEL_LINGAUSS,
    "SMCB_MODEL_GORDON": _lib.MODEL_GORDON, "SMCB_MODEL_THETALOGISTIC": _lib.MODEL_THETALOGISTIC,
    "SMCB_MODEL_BEARINGS": _lib.MODEL_BEARINGS, "SMCB_MODEL_MVLINGAUSS": _lib.MODEL_MVLINGAUSS,
    "SMCB_MODEL_DISCRETECOX": _lib.MODEL_DISCRETECOX, "SMCB_MODEL_STOCHVOLLEV": _lib.MODEL_STOCHVOLLEV,
    "SMCB_MAX_PARAMS": _lib.SMCB_MAX_PARAMS, "SMCB_SUMMARY_STRIDE": _lib.SUMMARY_STRIDE,
    "SMCB_SMOOTH_ON2": _lib.SMOOTH_ON2, "SMCB_SMOOTH_MCMC": _lib.SMOOTH_MCMC, "SMCB_SMOOTH_REJECT": _lib.SMOOTH_REJECT,
    "SMCB_SMOOTH_GATHER": _lib.SMOOTH_GATHER,
    "SMCB_ONLINE_PARIS": _lib.ONLINE_PARIS, "SMCB_ONLINE_ON2_W": _lib.ONLINE_ON2_W,
    "SMCB_ONLINE_PHI_PARIS": _lib.ONLINE_PHI_PARIS, "SMCB_ONLINE_PHI_ON2": _lib.ONLINE_PHI_ON2,
    "SMCB_TF_ON2_ROWS": _lib.TF_ON2_ROWS, "SMCB_TF_ON_LOGW": _lib.TF_ON_LOGW,
    "SMCB_VAR_EVE": _lib.VAR_EVE, "SMCB_VAR_SUMS": _lib.VAR_SUMS,
    "SMCB_VAR_CENTRED": _lib.VAR_CENTRED, "SMCB_VAR_WEIGHTS": _lib.VAR_WEIGHTS,
    "SMCB_BATCH_AUTO": _lib.BATCH_AUTO, "SMCB_BATCH_RESIDENT": _lib.BATCH_RESIDENT,
    "SMCB_BATCH_STREAMING": _lib.BATCH_STREAMING,
    "SMCB_BANK_STATE": _lib.BANK_STATE,
    "SMCB_CSMC_GENEALOGY": _lib.CSMC_GENEALOGY, "SMCB_CSMC_BACKWARD": _lib.CSMC_BACKWARD,
    "SMCB_HMM_MAX_K": _lib.HMM_MAX_K, "SMCB_HMM_FORWARD": _lib.HMM_FORWARD, "SMCB_HMM_BACKWARD": _lib.HMM_BACKWARD,
    "SMCB_HMM_SAMPLE": _lib.HMM_SAMPLE,
    "SMCB_KALMAN_MAX_D": _lib.KALMAN_MAX_D, "SMCB_KALMAN_FILTER": _lib.KALMAN_FILTER,
    "SMCB_KALMAN_SMOOTH": _lib.KALMAN_SMOOTH,
}
# integer #defines the Python side deliberately has no value for
NOT_MIRRORED = ()

# C type of a scalar parameter or return value -> its kind; every pointer or array is "pointer"
C_KINDS = {"int": "i32", "int32_t": "i32", "int64_t": "i64", "uint64_t": "u64", "double": "f64"}
CTYPES_KINDS = {C.c_int32: "i32", C.c_int64: "i64", C.c_uint64: "u64", C.c_double: "f64"}


# ------------------------------------------------------------------------------------------------------ the header
def _strip_comments(src):
    return re.sub(r"/\*.*?\*/", " ", src, flags=re.S)


def _code(src):
    """The header without comments and preprocessor lines."""
    return re.sub(r"^\s*#.*$", "", _strip_comments(src), flags=re.M)


def c_structs(src):
    """{struct name: [field names in declaration order]} of every `typedef struct { ... } name;`."""
    return {name: [re.search(r"(\w+)\s*(\[[^\]]*\])?$", d.strip()).group(1)
                   for decl in body.split(";") if decl.strip() for d in decl.split(",")]
            for body, name in re.findall(r"typedef\s+struct\s*\{([^{}]*)\}\s*(\w+)\s*;", _strip_comments(src))}


def c_prototypes(src):
    """{name: (return type, [parameter declarations])} of every smcb_* function the header declares."""
    out = {}
    for stmt in _code(src).split(";"):
        m = re.fullmatch(r"\s*(.*?)\b(smcb_\w+)\s*\((.*)\)\s*", re.split(r"[{}]", stmt)[-1], flags=re.S)
        if m:
            args = [a.strip() for a in m.group(3).split(",")]
            out[m.group(2)] = (m.group(1).strip(), [] if args == ["void"] else args)
    return out


def c_defines(src):
    """{name: value} of every `#define SMCB_<NAME> <value>`; a value that is not an integer raises."""
    return {name: int(value.strip().strip("()"))
            for name, value in re.findall(r"^\s*#\s*define\s+(SMCB_\w+)[ \t]+([^/\n]+)", src, flags=re.M)}


def compiled_layouts(structs):
    """{struct: (sizeof, [(field, offsetof, sizeof of the field)])}, printed by one C probe compiled against the
    header."""
    lines = []
    for s, fields in structs.items():
        lines.append(f'printf("{s} * 0 %zu\\n", sizeof({s}));')
        lines += [f'printf("{s} {f} %zu %zu\\n", offsetof({s}, {f}), sizeof((({s} *)0)->{f}));' for f in fields]
    src = "#include <stddef.h>\n#include <stdio.h>\n#include \"smcb.h\"\nint main(void) {\n%s\nreturn 0;\n}\n" % (
        "\n".join(lines))
    exe = os.path.join(ROOT, "oracle", "_build", "abi_probe")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    subprocess.run(["gcc", "-Wall", "-Werror", "-x", "c", "-", "-I", os.path.join(ROOT, "include"), "-o", exe],
                   input=src, text=True, check=True)
    out = {s: [None, []] for s in structs}
    for line in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines():
        s, f, off, size = line.split()
        if f == "*":
            out[s][0] = int(size)
        else:
            out[s][1].append((f, int(off), int(size)))
    return {s: tuple(v) for s, v in out.items()}


# ------------------------------------------------------------------------------------------------- the comparisons
def layout_mismatches(cls, size, fields):
    """What differs between a ctypes Structure and the compiler's layout of its C struct."""
    bad = []
    names = [f[0] for f in cls._fields_]
    if names != [f for f, _, _ in fields]:
        bad.append(f"{cls.__name__}: fields {names}, C has {[f for f, _, _ in fields]}")
    mine = {n: getattr(cls, n) for n in names}
    for f, off, sz in fields:
        if f in mine and (mine[f].offset, mine[f].size) != (off, sz):
            bad.append(f"{cls.__name__}.{f}: offset {mine[f].offset} size {mine[f].size}, C has {off} and {sz}")
    if C.sizeof(cls) != size:
        bad.append(f"{cls.__name__}: size {C.sizeof(cls)}, C has {size}")
    return bad


def c_kind(decl):
    """(kind, mirrored class of the struct pointed to or None) of a C parameter declaration or return type."""
    if "*" in decl or "[" in decl:
        return "pointer", STRUCTS.get(re.sub(r"\bconst\b|\*|\[[^\]]*\]", " ", decl).split()[0])
    t = [w for w in decl.split() if w != "const"][0]
    return C_KINDS.get(t, "unknown C type " + t), None


def ctypes_kind(t):
    if issubclass(t, C._Pointer):
        return "pointer", t._type_ if issubclass(t._type_, C.Structure) else None
    if t in (C.c_void_p, C.c_char_p):
        return "pointer", None
    return CTYPES_KINDS.get(t, "unknown ctypes type " + t.__name__), None


def prototype_mismatches(decls, prototypes):
    """What differs between (restype, argtypes) entries and the header's declarations: arity, return kind, argument
    kinds, and the struct behind every descriptor pointer."""
    bad = []
    for name, (res, args) in prototypes.items():
        if name not in decls:
            bad.append(f"{name}: not declared in the header")
            continue
        c_res, c_args = decls[name]
        if len(args) != len(c_args):
            bad.append(f"{name}: {len(args)} arguments, C has {len(c_args)}")
            continue
        for i, (t, c) in enumerate(zip([res] + args, [c_res] + c_args)):
            if ctypes_kind(t) != c_kind(c):
                what = "return value" if i == 0 else f"argument {i - 1}"
                bad.append(f"{name} {what}: {ctypes_kind(t)}, C has {c!r} {c_kind(c)}")
    return bad


def constant_mismatches(defines, mirror, not_mirrored):
    """Header #defines that are unclassified, classified twice, missing from the header, or mirrored unequal."""
    bad = [f"{n}: neither mirrored nor listed as not mirrored" for n in defines
           if n not in mirror and n not in not_mirrored]
    bad += [f"{n}: both mirrored and listed as not mirrored" for n in mirror if n in not_mirrored]
    bad += [f"{n}: not #defined in the header" for n in (*mirror, *not_mirrored) if n not in defines]
    bad += [f"{n}: header {defines[n]}, Python {v}" for n, v in mirror.items() if n in defines and defines[n] != v]
    return bad


# ------------------------------------------------------------------------------------------------------- the tests
@pytest.fixture(scope="module")
def layouts():
    return compiled_layouts(c_structs(HEADER))


@pytest.fixture(scope="module")
def lib():
    from particles_b200 import build
    build.build()
    return _lib.load()


def test_struct_table_covers_header_and_lib():
    assert sorted(c_structs(HEADER)) == sorted(STRUCTS)
    classes = {v for v in vars(_lib).values() if isinstance(v, type) and issubclass(v, C.Structure)}
    assert classes == set(STRUCTS.values())


def test_descriptor_layouts_match_compiler(layouts):
    assert sorted(layouts) == sorted(STRUCTS)
    bad = [b for s, cls in STRUCTS.items() for b in layout_mismatches(cls, *layouts[s])]
    assert not bad, "\n".join(bad)


def test_descriptors_reject_unknown_fields():
    """__slots__ = (): a misspelt field raises instead of becoming a Python attribute the library never reads."""
    for cls in STRUCTS.values():
        assert vars(cls).get("__slots__") == (), cls.__name__
        with pytest.raises(AttributeError):
            cls().not_a_field = 1
        with pytest.raises(AttributeError):
            cls(not_a_field=1)


def test_prototypes_match_header():
    decls = c_prototypes(HEADER)
    assert len(decls) == len(re.findall(r"\bsmcb_\w+\s*\(", _code(HEADER)))     # the parse skipped no declaration
    assert set(_lib.PROTOTYPES) == set(decls)
    bad = prototype_mismatches(decls, _lib.PROTOTYPES)
    assert not bad, "\n".join(bad)


def test_constants_match_header():
    bad = constant_mismatches(c_defines(HEADER), CONSTANTS, NOT_MIRRORED)
    assert not bad, "\n".join(bad)


def test_library_exports_every_declared_symbol(lib):
    syms = sorted(c_prototypes(HEADER))
    assert len(syms) >= 25
    raw = C.CDLL(_lib.SO_PATH)
    for s in syms:
        assert hasattr(raw, s), f"{s} declared in include/smcb.h but not exported"
    assert set(_lib.PROTOTYPES) == set(syms)          # the ctypes layer binds exactly the header
    assert lib.smcb_version() == 100
    assert lib.smcb_resample_scratch_doubles(1000, 500) >= 1000 + 500


# ------------------------------------------------------------------------------------- the checker on broken mirrors
def test_layout_check_reports_swapped_fields(layouts):
    fields = list(_lib.HmmDesc._fields_)
    fields[1], fields[2] = fields[2], fields[1]           # K (int32_t) and B (int64_t)

    class Swapped(C.Structure):
        _fields_ = fields

    bad = layout_mismatches(Swapped, *layouts["smcb_hmm_desc"])
    assert bad[0].startswith("Swapped: fields ['method', 'B', 'K', "), bad
    assert "Swapped.K: offset 16 size 4, C has 4 and 4" in bad, bad


def test_prototype_check_reports_wrong_kinds():
    decls = c_prototypes(HEADER)
    assert _lib.PROTOTYPES["smcb_filter_step"] == (C.c_int, [C.c_void_p, C.c_int64])
    broken = {"smcb_filter_step": (C.c_int, [C.c_void_p, C.c_int]),                   # int in place of int64_t
              "smcb_hmm": (C.c_int, [C.c_void_p, C.POINTER(_lib.KalmanDesc)]),        # the wrong descriptor
              "smcb_uniform": (C.c_int, [C.c_void_p, C.c_void_p])}                   # one argument short
    bad = prototype_mismatches(decls, broken)
    assert len(bad) == 3, bad
    assert bad[0].startswith("smcb_filter_step argument 1: ('i32', None), C has 'int64_t nsteps'"), bad
    assert bad[1].startswith("smcb_hmm argument 1: ('pointer', <class 'particles_b200._lib.KalmanDesc'>)"), bad
    assert bad[2] == "smcb_uniform: 2 arguments, C has 3", bad


def test_constant_check_reports_unequal_and_unclassified():
    defines = c_defines(HEADER)
    off_by_one = dict(CONSTANTS, SMCB_RS_SSP=CONSTANTS["SMCB_RS_SSP"] + 1)
    assert "SMCB_RS_SSP: header 4, Python 5" in constant_mismatches(defines, off_by_one, NOT_MIRRORED)
    unclassified = dict(defines, SMCB_NEW=7)
    assert "SMCB_NEW: neither mirrored nor listed as not mirrored" in \
        constant_mismatches(unclassified, CONSTANTS, NOT_MIRRORED)
