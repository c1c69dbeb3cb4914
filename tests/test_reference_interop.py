"""Wire compatibility with the UNMODIFIED reference package (CPU).

``tests/golden/reference_wire.json`` holds messages recorded from pytensor-federated 1.0.2: the
``InputArrays`` its client sends for fixed inputs (hex), and its ``ArraysToArraysService``'s reply to
them for ``f(a, b) = -(a - 1)^2 - sum((b + 2)^2)`` with ``wrap_logp_grad_func``.  The golden tests
check this package against those bytes and need nothing outside the repository.

The live tests additionally start the reference's own service and client; they need
``baseline/_ref`` (``pip install --no-deps --target`` of a reference checkout, git-ignored), whose
missing third-party imports (betterproto, grpclib) are satisfied by ``baseline/shims``.
"""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from _helpers import ServerProcess, free_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "baseline", "_ref")
SHIMS = os.path.join(ROOT, "baseline", "shims")

GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_wire.json")
GOLDEN_INPUTS = {
    "ints": [np.array(6), np.array(7)],
    "scalar_vector": [np.array(3.0), np.array([0.0, 1.0])],
}

pytestmark = pytest.mark.timeout(180)
needs_reference = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "pytensor_federated")),
                                     reason="reference not installed")


def _golden():
    import json

    with open(GOLDEN) as fh:
        return {k: {kk: (bytes.fromhex(v) if kk in ("request", "reply") else v) for kk, v in rec.items()}
                for k, rec in json.load(fh).items()}


def _f(a, b):
    return np.asarray(-(a - 1.0) ** 2 - np.sum((b + 2.0) ** 2)), [np.asarray(-2 * (a - 1.0)), -2 * (b + 2.0)]


@pytest.mark.parametrize("case", sorted(GOLDEN_INPUTS))
def test_reference_requests_decode_here(case):
    from pytensor_federated_b200.rpc import InputArrays

    msg = InputArrays.FromString(_golden()[case]["request"])
    got = msg.arrays   # the decoding path the service uses
    assert msg.uuid == f"uuid-{case}"
    for g, want in zip(got, GOLDEN_INPUTS[case], strict=True):
        assert g.dtype == want.dtype and g.shape == want.shape
        np.testing.assert_array_equal(g, want)


@pytest.mark.parametrize("case", ["ints", "scalar_vector"])
def test_requests_encode_byte_identical_to_the_reference(case):
    from pytensor_federated_b200.rpc import encode_arrays_message

    assert encode_arrays_message(GOLDEN_INPUTS[case], uuid=f"uuid-{case}") == _golden()[case]["request"]


@pytest.mark.parametrize("case", ["ints", "scalar_vector"])
def test_service_replies_like_the_reference_service(case):
    from pytensor_federated_b200 import ArraysToArraysService, wrap_logp_grad_func
    from pytensor_federated_b200.npproto.utils import ndarray_to_numpy
    from pytensor_federated_b200.rpc import InputArrays, OutputArrays
    from pytensor_federated_b200.service import get_useful_event_loop

    gold = _golden()[case]
    svc = ArraysToArraysService(wrap_logp_grad_func(_f))
    reply = get_useful_event_loop().run_until_complete(svc.evaluate(InputArrays.FromString(gold["request"])))
    ours = OutputArrays.FromString(bytes(reply))
    theirs = OutputArrays.FromString(gold["reply"])
    assert ours.uuid == theirs.uuid == f"uuid-{case}"
    for a, b, want in zip(ours.items, theirs.items, gold["reply_arrays"], strict=True):
        a, b = ndarray_to_numpy(a), ndarray_to_numpy(b)
        assert a.dtype == b.dtype and a.shape == b.shape
        np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(b, want)


def _ref_env():
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([SHIMS, REF, ROOT])
    return env


REF_SERVER = textwrap.dedent(
    """
    import asyncio, sys
    import numpy as np
    import grpclib.server
    from pytensor_federated import ArraysToArraysService, wrap_logp_grad_func

    def f(a, b):
        return np.asarray(-(a - 1.0) ** 2 - np.sum((b + 2.0) ** 2)), [np.asarray(-2 * (a - 1.0)), -2 * (b + 2.0)]

    async def main(port):
        server = grpclib.server.Server([ArraysToArraysService(wrap_logp_grad_func(f))])
        await server.start("127.0.0.1", port)
        print("READY", flush=True)
        await server.wait_closed()

    asyncio.new_event_loop().run_until_complete(main(int(sys.argv[1])))
    """
)

REF_CLIENT = textwrap.dedent(
    """
    import sys
    import numpy as np
    from pytensor_federated import ArraysToArraysServiceClient
    client = ArraysToArraysServiceClient("127.0.0.1", int(sys.argv[1]))
    out = client.evaluate(np.array(6), np.array(7))
    assert out[0] == 42, out
    out = client.evaluate(np.array(1.5), np.array(4.0), use_stream=False)
    assert float(out[0]) == 6.0, out
    print("OK", flush=True)
    """
)


@needs_reference
def test_product_client_talks_to_reference_server():
    from pytensor_federated_b200 import LogpGradServiceClient, service

    port = free_port()
    proc = subprocess.Popen([sys.executable, "-c", REF_SERVER, str(port)], env=_ref_env(), stdout=subprocess.PIPE, text=True)
    try:
        assert proc.stdout.readline().strip() == "READY"
        client = LogpGradServiceClient("127.0.0.1", port)
        logp, (da, db) = client.evaluate(np.array(3.0), np.array([0.0, 1.0]))
        assert logp == -(2.0**2) - (4.0 + 9.0)
        assert da == -4.0
        np.testing.assert_array_equal(db, [-4.0, -6.0])
        load = service.get_useful_event_loop().run_until_complete(service.get_load_async("127.0.0.1", port))
        assert load.n_clients == 1 and 0 < load.percent_ram < 100
        del client
    finally:
        proc.terminate()
        proc.wait(10)


@needs_reference
def test_reference_client_talks_to_product_server():
    with ServerProcess() as server:
        res = subprocess.run(
            [sys.executable, "-c", REF_CLIENT, str(server.port)], env=_ref_env(), capture_output=True, text=True, timeout=120
        )
        assert res.returncode == 0, res.stderr[-2000:]
        assert "OK" in res.stdout
