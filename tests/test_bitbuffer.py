"""The host bit buffer's write protocol (jsmpeg_b200/csrc/bitbuffer.h, compiled into the product by
engine.cu) on the CPU under AddressSanitizer: the returned pointer always covers the requested bytes
(the reference's own sizing does not: src/wasm/buffer.c:53-57 -- advisor finding of round 1), and the
state equals the compiled reference's wherever the reference stays inside its allocation
(stored in tests/golden/reference/bitbuffer.npy by tools/make_golden.py)."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def test_write_protocol_under_asan_and_against_the_reference():
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not asan or not os.path.exists(asan):
        pytest.skip("libasan not available")
    lib = os.path.join(HERE, "emu", "libbitbuffer_test_asan.so")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-shared", "-fPIC", "-fsanitize=address", "-fno-omit-frame-pointer",
                           "-o", lib, os.path.join(HERE, "emu", "bitbuffer_test.cpp")])
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([sys.executable, os.path.join(HERE, "emu", "bitbuffer_check.py"), lib,
                        os.path.join(HERE, "golden", "reference", "bitbuffer.npy")], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "bitbuffer ok" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
