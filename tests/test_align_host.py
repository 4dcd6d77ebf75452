"""glic_mapper_align without a GPU: the ctypes structs against the header's layout (compiled with the system C compiler), and the
NULL-mapper rejection."""
import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _c_layout(tmp_path, struct, fields):
    """[sizeof, offsetof(field)...] of a header struct, as a C compiler lays it out"""
    src = tmp_path / ("%s.c" % struct)
    body = "".join('    printf(" %%zu", offsetof(%s, %s));\n' % (struct, f) for f in fields)
    src.write_text('#include "glic_b200.h"\n#include <stddef.h>\n#include <stdio.h>\nint main(void) {\n'
                   '    printf("%%zu", sizeof(%s));\n%s    printf("\\n");\n    return 0;\n}\n' % (struct, body))
    exe = tmp_path / struct
    r = subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]


def test_structs_match_the_header(tmp_path):
    from gaussian_lic_b200 import capi
    for py, name in ((capi.AlignParams, "glic_align_params"), (capi.AlignResult, "glic_align_result")):
        fields = [f for f, _ in py._fields_]
        want = _c_layout(tmp_path, name, fields)
        got = [C.sizeof(py)] + [getattr(py, f).offset for f in fields]
        assert got == want, (name, got, want)
        sizes = [getattr(py, f).size for f in fields]
        assert sum(sizes) == C.sizeof(py) == want[0]                   # no padding the header does not have either
    assert [f for f, _ in capi.AlignResult._fields_][:3] == ["R_wc", "t_wc", "E"]
    assert capi.AlignResult.steps.offset == C.sizeof(capi.AlignResult) - 8


def test_null_mapper_is_rejected_without_a_device():
    from gaussian_lic_b200 import capi
    p = capi.AlignParams(10, 1e-3, 1e-3, 0.0, 0)
    r = capi.AlignResult()
    r.steps = 1234
    assert capi.lib.glic_mapper_align(None, 0, 0, C.byref(p), C.byref(r), None) == -1
    assert b"null" in capi.lib.glic_last_error()
    assert r.steps == 1234                                              # nothing written
    assert capi.lib.glic_mapper_align(None, 0, 0, None, None, None) == -1
