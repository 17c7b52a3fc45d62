"""CPU: the C-ABI library loads, exports every symbol include/step_b200.h declares and reads no environment variable; the
ctypes binding read from the header has the C compiler's struct layouts and constants, and its reader refuses what it
cannot read; the product never imports the oracle; no compute calls are made here (no GPU in this tier)."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "step_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(step_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from step_b200 import _lib
    lib = _lib.lib()
    declared = header_symbols()
    assert len(declared) >= 25
    for name in declared:
        assert hasattr(lib, name), "libstep_b200.so does not export %s" % name
    assert lib.step_version() == 100
    # the python binding is the header's
    assert _lib.exported_symbols() == declared


def test_library_is_sm90a_native():
    out = subprocess.run(["cuobjdump", "-lelf", os.path.join(ROOT, "step_b200", "libstep_b200.so")],
                         capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_library_reads_no_environment():
    """A call's result and speed follow from its arguments alone: no object of the library calls getenv.  The objects are
    checked, not the .so, because the .so links cudart statically and cudart reads its own variables."""
    from step_b200 import build
    build.build()
    readers = []
    for src in build.SOURCES:
        obj = os.path.join(build.OBJ, src.replace(".cu", ".o"))
        out = subprocess.run(["nm", "--undefined-only", obj], capture_output=True, text=True, check=True).stdout
        readers += ["%s: %s" % (src, s) for s in out.split() if s in ("getenv", "secure_getenv")]
    assert not readers, readers


def test_product_never_touches_the_oracle():
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "step_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                if re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M) or "oracle/" in txt or "/root/reference" in txt:
                    bad.append(os.path.join(dirpath, f))
    assert not bad, bad


def test_ops_raise_without_cuda_tensor():
    import pytest
    import torch
    from step_b200 import roi_layers
    x = torch.zeros(1, 8, 4, 4)
    with pytest.raises(RuntimeError):
        roi_layers.roi_align(x, torch.zeros(1, 5), (7, 7), 1 / 16., 0)
    assert roi_layers.nms(torch.zeros(0, 4), torch.zeros(0), 0.4).numel() == 0  # empty in -> empty out, nms.h:41


def test_argument_errors_are_reported_before_any_device_work():
    """The entry points validate their arguments first (STEP_E_ARG + step_last_error text), the role AT_ASSERTM plays in
    the reference's ops: checked here without a GPU on the fused bottleneck exit, which exists for the reference's head
    widths only (two_branch.py:190-192)."""
    from step_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_char * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    rc = lib.step_bottleneck_exit_f16(p, 128, p, p, 1024, p, None, 1, None, 0, p, 256, 64, 128, 1024, 256, None)
    assert rc == _lib.E_ARG
    assert b"planes 256" in lib.step_last_error()
    rc = lib.step_bottleneck_exit_f16(None, 256, p, p, 1024, p, None, 1, None, 0, p, 256, 64, 256, 1024, 256, None)
    assert rc == _lib.E_ARG and b"null pointer" in lib.step_last_error()


def test_binding_matches_the_c_compiler(tmp_path):
    """Every struct the binding reads from the header has the host C compiler's size and the offset and size of every
    field, and every enum constant its value."""
    from step_b200 import _lib
    lines, want = [], {}
    for name, cls in _lib.STRUCTS.items():
        lines.append('printf("%s %%zu\\n", sizeof(%s));' % (name, name))
        want[name] = "%d" % ctypes.sizeof(cls)
        for f, _ in cls._fields_:
            lines.append('printf("%s.%s %%zu %%zu\\n", offsetof(%s, %s), sizeof(((%s*)0)->%s));' % (name, f, name, f, name, f))
            want["%s.%s" % (name, f)] = "%d %d" % (getattr(cls, f).offset, getattr(cls, f).size)
    for name, value in _lib.CONSTANTS.items():
        lines.append('printf("%s %%lld\\n", (long long)%s);' % (name, name))
        want[name] = "%d" % value
    src = tmp_path / "probe.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "step_b200.h"\nint main(void) {\n%s\nreturn 0;\n}\n'
                   % "\n".join(lines))
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "probe")], check=True)
    out = subprocess.run([str(tmp_path / "probe")], capture_output=True, text=True, check=True).stdout
    got = dict(line.split(" ", 1) for line in out.splitlines())
    assert got == want


@pytest.mark.parametrize("decl, name", [
    ("int step_f(void (*done)(int), step_stream_t stream);", "done"),     # function-pointer parameter
    ("int step_f(double x);", "double x"),                                # scalar type it does not know
    ("int step_f(step_s s);", "step_s s"),                                # struct passed by value
    ("unsigned step_f(void);", "unsigned step_f"),                        # result type it does not know
    ("enum { STEP_X = 1, STEP_Y };", "STEP_Y"),                           # implicit enum value
    ("enum { STEP_X = 1 + 2 };", "STEP_X"),                               # value expression it does not evaluate
    ("typedef struct { int a; short b; } step_t;", "short b"),            # field type it does not know
    ("typedef struct { int a[STEP_N]; } step_t;", "STEP_N"),              # array length it does not know
    ("struct step_t { int a; };", "struct step_t"),                       # declaration form it does not know
])
def test_header_reader_refuses_what_it_cannot_read(decl, name):
    from step_b200 import _lib
    ok = "typedef struct { int a; } step_s;\n"
    with pytest.raises(ValueError, match=re.escape(name)):
        _lib.read_header(ok + decl)
