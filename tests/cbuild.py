"""Builds the tests' native helpers: the C oracles (tests/*_oracle.c) as shared objects loaded through ctypes, and the C++ API mirrors
(tests/cpp/*.cc) as executables linked against the product library.

An oracle's shared object is cached under the temporary directory, named by uid and key(); the tree is never written.  The key covers
the compiler command and every file the build reads from the tree, so an edit to any of them, included files too, rebuilds it."""
import ctypes
import hashlib
import os
import re
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_INCLUDE = re.compile(rb'^[ \t]*#[ \t]*include[ \t]*"([^"]+)"', re.M)
_loaded = {}


def _command():
    return [os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-std=gnu11", "-ffp-contract=off", "-fno-fast-math", "-shared"]


def _reached(path, seen):
    """Appends `path` and, depth first, every existing file it reaches through #include "...", each resolved relative to the file
    that includes it (a quoted name not found there is a system header, which the compiler resolves)."""
    path = os.path.realpath(path)
    if path not in seen and os.path.isfile(path):
        seen.append(path)
        with open(path, "rb") as f:
            for name in _INCLUDE.findall(f.read()):
                _reached(os.path.join(os.path.dirname(path), name.decode()), seen)
    return seen


def key(*sources):
    """Hash of the compiler command, the C files `sources` (paths) and every file they reach through #include "..."."""
    h = hashlib.sha1("\0".join(_command() + ["-lm"]).encode())
    seen = []
    for s in sources:
        _reached(s, seen)
    for p in seen:
        with open(p, "rb") as f:
            data = f.read()
        h.update(b"%d\0" % len(data) + data)
    return h.hexdigest()[:16]


def load(*sources):
    """ctypes.CDLL of the tests/ C files `sources` compiled together into one shared object; built at most once per key and loaded at
    most once per process."""
    paths = [os.path.join(HERE, s) for s in sources]
    k = key(*paths)
    if k not in _loaded:
        stem = os.path.splitext(sources[0])[0]
        so = os.path.join(tempfile.gettempdir(), f"b200_{stem}_{os.getuid()}_{k}.so")
        if not os.path.exists(so):
            tmp = so + f".{os.getpid()}.tmp"
            subprocess.check_call(_command() + ["-o", tmp] + paths + ["-lm"])
            os.replace(tmp, so)
        _loaded[k] = ctypes.CDLL(so)
    return _loaded[k]


def cpp_mirror(name, out_dir):
    """Builds tests/cpp/<name>.cc against include/ and the product library; returns the executable's path."""
    from stella_vslam_b200 import build as builder
    lib = builder.build()
    exe = os.path.join(str(out_dir), name)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), os.path.join(HERE, "cpp", name + ".cc"),
                           "-o", exe, lib, "-Wl,-rpath," + os.path.dirname(lib), "-ldl", "-lpthread", "-lrt"])
    return exe
