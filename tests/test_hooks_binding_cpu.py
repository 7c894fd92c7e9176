"""CPU checks of the test hooks' binding: the library's exported mlease_internal_* symbols, the prototypes of
ml-ease_b200/csrc/mlease_internal.h and the ctypes table of mlease_b200/_hooks.py are one set and agree argument by argument;
StageCtrl, which the Newton hooks copy byte for byte, has the same layout in C and in numpy; and no test or tool binds a hook
on its own.  A drifted signature or offset would hand the kernels wrong pointers."""
import ctypes as C
import glob
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ml-ease_b200", "csrc")
HEADER = os.path.join(CSRC, "mlease_internal.h")


def _prototypes():
    """name -> list of (type, is_pointer) of every hook the header declares"""
    src = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)
    out = {}
    for name, args in re.findall(r"\bint\s+(mlease_internal_\w+)\s*\(([^)]*)\)\s*;", src):
        params = []
        for a in args.split(","):
            a = a.strip()
            ptr = "*" in a
            base = re.sub(r"\bconst\b", "", a.split("*")[0]).split()[0]
            params.append((base, ptr))
        out[name] = params
    return out


def _exported():
    from mlease_b200 import build
    so = build.build()
    syms = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True, check=True).stdout
    return set(re.findall(r"\b(mlease_internal_\w+)\b", syms))


def test_exports_header_and_table_are_one_set_of_18():
    """The 18 hooks, the two partition read-backs (partition_info, partition_data) included."""
    from mlease_b200 import _hooks
    declared = set(_prototypes())
    assert len(declared) == 18, sorted(declared)
    assert _exported() == declared, sorted(_exported() ^ declared)
    assert set(_hooks.SIG) == declared, sorted(set(_hooks.SIG) ^ declared)


def test_table_matches_the_prototypes():
    """Width and pointer-ness of every argument: int32_t -> c_int32, int64_t -> c_int64, a pointer -> c_void_p or POINTER(...)."""
    from mlease_b200 import _hooks
    scalars = {"int32_t": C.c_int32, "int64_t": C.c_int64}
    for name, params in _prototypes().items():
        table = _hooks.SIG[name]
        assert len(table) == len(params), (name, len(table), len(params))
        for i, ((base, is_ptr), t) in enumerate(zip(params, table)):
            if is_ptr:
                assert t is C.c_void_p or issubclass(t, C._Pointer), (name, i, base, t)
            else:
                assert t is scalars[base], (name, i, base, t)


def test_stage_ctrl_layout(tmp_path):
    """The header compiles as pedantic C99, and sizeof / every offsetof of StageCtrl equal STAGE_CTRL's itemsize and offsets."""
    from mlease_b200 import _hooks
    names = _hooks.STAGE_CTRL.names
    src = tmp_path / "stage.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "mlease_internal.h"\nint main(void) {\n'
                   '  printf("%zu\\n", sizeof(StageCtrl));\n' +
                   "".join('  printf("%%zu\\n", offsetof(StageCtrl, %s));\n' % n for n in names) + "  return 0;\n}\n")
    exe = str(tmp_path / "stage")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", CSRC, "-o", exe, str(src)])
    got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert got[0] == _hooks.STAGE_CTRL.itemsize, (got[0], _hooks.STAGE_CTRL.itemsize)
    want = [_hooks.STAGE_CTRL.fields[n][1] for n in names]
    assert got[1:] == want, [(n, g, w) for n, g, w in zip(names, got[1:], want) if g != w]


def test_no_test_or_tool_binds_a_hook():
    """argtypes of a hook are set in _hooks.bound() only: not on the hook's attribute, nor on a name a hook was assigned to."""
    hits = []
    for path in glob.glob(os.path.join(ROOT, "tests", "**", "*.py"), recursive=True) + glob.glob(os.path.join(ROOT, "tools", "*.py")):
        txt = open(path).read()
        hook_names = set(re.findall(r"\b(\w+)\s*=\s*[^\n=]*\bmlease_internal_\w+", txt))
        for line in txt.splitlines():
            for target in re.findall(r"([\w.]+)\s*\.\s*argtypes\b", line):
                if "mlease_internal_" in target or target in hook_names:
                    hits.append("%s: %s" % (os.path.relpath(path, ROOT), line.strip()))
    assert not hits, hits
