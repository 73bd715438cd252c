"""The device frame writer's tests (test_frame_encode_dev.py) on a box without a GPU: against the emulator build of the whole
library (tests/simt/build_sim_library.sh), with 1 MiB chunks so that small calls still cross chunk boundaries."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def sim_library():
    subprocess.run(["bash", os.path.join(HERE, "simt", "build_sim_library.sh")], check=True, capture_output=True)
    return os.path.join(HERE, "simt", "_build", "libb200lz4_sim.so")


def test_device_frame_writer_on_the_emulator_library(sim_library):
    env = dict(os.environ, B200LZ4_TEST_SO=sim_library, B200LZ4_CHUNK_MB="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_frame_encode_dev.py"), "-m", "gpu", "-q", "-x",
                        "-p", "no:cacheprovider", "-W", "ignore::DeprecationWarning"],
                       env=env, cwd=os.path.dirname(HERE), capture_output=True, text=True)
    assert r.returncode == 0 and "7 passed" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
