import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def fds_bytes():
    with open(os.path.join(ROOT, "tests", "golden", "schemas.binpb"), "rb") as fh:
        return fh.read()


@pytest.fixture(scope="session")
def oracle(fds_bytes):
    import orc
    return orc.Schema(fds_bytes)


@pytest.fixture(scope="session")
def hsim(fds_bytes):
    import hostsim
    return hostsim.Schema(fds_bytes)


# every GPU test runs against each kernel path: the default (lock-step kernels in front of the
# per-thread kernels on both sides), the per-thread kernels alone, the lock-step request side only
_ENGINE_PATHS = {
    # everything through the lock-step kernels first (the size routing would send the small test items
    # straight to the per-thread kernels)
    "default": {"GGR_LOCKSTEP_MIN_BYTES": "0"},
    "size_routing": {},
    "per_thread": {"GGR_COOP_ENC": "0", "GGR_COOP": "0"},
    # the one-lane-per-object walker of round 1 in place of the token-parallel one (still the request-body path)
    "old_walker": {"GGR_WALK": "0", "GGR_LOCKSTEP_MIN_BYTES": "0"},
    "lockstep_request_only": {"GGR_COOP": "0", "GGR_LOCKSTEP_MIN_BYTES": "0"},
    # host entry points cut into many small chunks over two slots: exercises the copy/compute pipeline
    "small_chunks": {"GGR_CHUNK_ITEMS": "128", "GGR_SLOTS": "2", "GGR_LOCKSTEP_MIN_BYTES": "0"},
    # chunks cut by the byte budget, short chunks at both ends of a batch (the ramp needs chunks of at least 512 items and
    # four of them), issuing threads asleep on blocking events instead of spinning
    "ramped_chunks": {"GGR_CHUNK_ITEMS": "512", "GGR_CHUNK_BYTES": "400000", "GGR_SLOTS": "3", "GGR_BLOCKING_SYNC": "1"},
    # every call leaves its scratch buffers full of well-formed stale records (IR nodes, sizes, list entries): a kernel
    # that reads a slot nobody wrote in the current call shows up as wrong bytes (round 2: null members in the walker)
    "poisoned": {"GGR_POISON": "1", "GGR_LOCKSTEP_MIN_BYTES": "0"},
    "poisoned_size_routing": {"GGR_POISON": "1"},
}


@pytest.fixture(scope="session", params=list(_ENGINE_PATHS))
def engine(request):
    import ggrmcp_b200
    env = _ENGINE_PATHS[request.param]
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        e = ggrmcp_b200.Engine(0)  # the engine reads its switches at creation
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    yield e
    e.close()


@pytest.fixture(scope="session")
def schema(engine, fds_bytes):
    return engine.register(fds_bytes)
