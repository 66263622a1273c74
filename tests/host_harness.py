"""Builds a host harness under tests/cpp into a shared library for one test module.  Test infrastructure only."""
import ctypes as C
import os
import subprocess

CPP = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp")


def build_harness(tmp_path_factory, name, *flags):
    """tests/cpp/<name>.cpp built by g++ -std=c++17 -O2 with these extra flags into a shared library in a new pytest temp dir; its
    CDLL"""
    so = str(tmp_path_factory.mktemp(name) / (name + ".so"))
    subprocess.check_call(["g++", "-std=c++17", "-O2", *flags, "-shared", "-fPIC", "-o", so, os.path.join(CPP, name + ".cpp")])
    return C.CDLL(so)
