"""In-tree build of the product's shared objects (nvcc, sm_90a).  No JIT cache: the .so files sit next to the
sources, so the package is importable from the repository tree."""
from __future__ import annotations

import os
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
LIB_QMM = os.path.join(PKG, "libb200qmm.so")
LIB_PLUGIN = os.path.join(PKG, "libggml-b200.so")
BACKEND = os.path.join(PKG, "backend")


def build_kernels(jobs: int = 8) -> str:
    subprocess.check_call(["make", "-s", f"-j{jobs}", "-C", os.path.join(PKG, "csrc")])
    return LIB_QMM


def build_plugin_objects(objdir: str, ref: str, jobs: int = 8) -> None:
    """The plugin's C++ objects compile against the reference's internal ggml headers: only where those sources exist."""
    subprocess.check_call(["make", "-s", f"-j{jobs}", "-C", BACKEND, "objs", f"OBJDIR={objdir}", f"REF={ref}"])


def link_plugin(objdir: str, hostlib: str, jobs: int = 8) -> str:
    """Compiles the kernels and links them with the plugin's C++ objects (objdir) against the host's libggml-base (hostlib)."""
    subprocess.check_call(["make", "-s", f"-j{jobs}", "-C", BACKEND, "link", f"OBJDIR={objdir}", f"HOSTLIB={hostlib}"])
    return LIB_PLUGIN
