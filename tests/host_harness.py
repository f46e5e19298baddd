"""Builds the host harnesses that compile the device headers for the CPU (tests/*_vs_oracle.cpp through tests/host_shim/), with the
flags every source test shares: IEEE binary32 in written order (-ffp-contract=off), or with contraction on to show that the comparison
notices a fused multiply-add."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")


def compile_harness(tmp_path, source, contract=False, link_oracle=False):
    """g++ tests/<source>.cpp into tmp_path; link_oracle links oracle/liboxc_oracle.so (built first when missing or stale)"""
    exe = str(tmp_path / (source + ("_fma" if contract else "")))
    cmd = ["g++", "-O2", "-std=c++17", "-Wno-unknown-pragmas"] + (["-mfma", "-ffp-contract=fast"] if contract else ["-ffp-contract=off"])
    cmd += ["-I", os.path.join(ROOT, "tests", "host_shim"), "-I", os.path.join(ROOT, "oxylus_b200", "csrc"),
            os.path.join(ROOT, "tests", source + ".cpp"), "-o", exe]
    if link_oracle:
        import pyoracle

        pyoracle.build()
        cmd += ["-L", ORACLE, "-loxc_oracle", f"-Wl,-rpath,{ORACLE}"]
    subprocess.check_call(cmd)
    return exe


def skip_without_fma():
    """the contraction checks need a host CPU with an FMA unit"""
    with open("/proc/cpuinfo") as f:
        if "fma" not in f.read():
            pytest.skip("host CPU has no FMA unit")
