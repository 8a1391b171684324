"""Runs one compiled drop-in test (tests/cpp/*dropin_test.cpp, built into oracle/_ref/ by oracle/ref_shim/Makefile where the
reference's sources are present at build time; elsewhere the test skips)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_dropin(name: str, ok_line: str, timeout: int = 600) -> None:
    """Runs oracle/_ref/<name> against limbo_b200/lib and asserts that it exits with 0 and prints ok_line."""
    binary = os.path.join(ROOT, "oracle", "_ref", name)
    if not os.path.exists(binary):
        pytest.skip(f"oracle/_ref/{name} not built (needs the reference's sources at build time)")
    env = dict(os.environ, LD_LIBRARY_PATH=os.path.join(ROOT, "limbo_b200", "lib") + ":" + os.environ.get("LD_LIBRARY_PATH", ""))
    r = subprocess.run([binary], capture_output=True, text=True, timeout=timeout, env=env)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and ok_line in r.stdout, r.stdout + r.stderr
