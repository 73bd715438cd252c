"""The incremental device LZ4Block writer's and reader's tests (test_lz4block_stream_dev.py) on a box without a GPU: against
the emulator build of the whole library.  The library is built here with the same sources and flags as
tests/simt/build_sim_library.sh, plus tests/simt/alloc_count.h force-included (which includes tests/simt/copy_count.h), so
that the tests can also count the bytes the library copies between host and device and the device memory it holds."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def counted_sim_library():
    out = os.path.join("tests", "simt", "_build")
    os.makedirs(os.path.join(ROOT, out), exist_ok=True)
    cxx = ["g++", "-O1", "-std=c++17", "-fPIC", "-Wno-unknown-pragmas", "-Wno-attributes", "-DB200_HOST_SIM", "-Itests/simt",
           "-Ilz4-java_b200/csrc", "-include", "tests/simt/alloc_count.h"]
    srcs = [("tests/simt/sim_launchers.cpp", []), ("tests/simt/copy_count.cpp", []),
            ("tests/simt/alloc_count.cpp", [])] + \
           [(f"lz4-java_b200/csrc/{f}.cu", ["-x", "c++"]) for f in ("capi", "frame", "containers")]
    objs = [os.path.join(out, "lz4block_stream_counted_" + os.path.basename(s).split(".")[0] + ".o") for s, _ in srcs]

    def compile_one(k):
        s, lang = srcs[k]
        return subprocess.run(cxx + lang + ["-c", s, "-o", objs[k]], cwd=ROOT, capture_output=True, text=True)

    with ThreadPoolExecutor(len(srcs)) as pool:
        for r in pool.map(compile_one, range(len(srcs))):
            assert r.returncode == 0, r.stderr[-3000:]
    so = os.path.join(out, "libb200lz4_sim_lz4block_stream_counted.so")
    r = subprocess.run(["g++", "-shared", "-o", so] + objs + ["-lpthread"], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return os.path.join(ROOT, so)


def test_incremental_lz4block_calls_on_the_emulator_library(counted_sim_library):
    env = dict(os.environ, B200LZ4_TEST_SO=counted_sim_library, B200LZ4_CHUNK_MB="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_lz4block_stream_dev.py"), "-m", "gpu", "-q", "-x",
                        "-p", "no:cacheprovider", "-W", "ignore::DeprecationWarning"],
                       env=env, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0 and "15 passed" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
