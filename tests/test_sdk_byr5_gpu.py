"""BYR5 through the unmodified SDK (integration/_build): ConvertBYR5ToFrame16s is interposed, the packed frame goes to the
GPU, and the encoded samples are byte-identical to the plain reference's."""
import json

import pytest

from test_sdk_integration_gpu import needs_build, run, shim_stats

pytestmark = pytest.mark.gpu


@needs_build
@pytest.mark.parametrize("size", [(2048, 1152), (1040, 544)])
def test_public_api_encode_byr5(size):
    """Sync loop and encoder pool: the same sample digests as the reference, no frame on the CPU transform.  1040 wide:
    plane rows of 520 samples, whose packed segments sit 8 and 4 bytes off 16-byte boundaries."""
    w, h = size
    gpu = run("sdk_roundtrip", w, h, 3, 2, 24, 0, "byr5")
    ref = run("sdk_roundtrip_ref", w, h, 3, 2, 24, 0, "byr5")
    g, r = json.loads(gpu.stdout.strip().splitlines()[-1]), json.loads(ref.stdout.strip().splitlines()[-1])
    assert g["format"] == "byr5"
    assert g["sample_bytes"] == r["sample_bytes"]
    assert g["sample_digest"] == r["sample_digest"] and g["pool_sample_digest"] == r["pool_sample_digest"]
    st = shim_stats(gpu.stderr)
    assert st["fwd_gpu"] >= 4 + 32 and st["fwd_ref"] == 0 and st["cuda_errors"] == 0
