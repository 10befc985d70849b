"""16-bit RGBA sources (B64A, RG64) through the unmodified SDK (integration/): CFHD_PIXEL_FORMAT_B64A / RG64 with
CFHD_ENCODED_FORMAT_RGB_444 or RGBA_4444.  The converter hooks record the packed frame, the GPU transforms all three or
four channels from it (the plan's descriptor carries CFB_FRAME_ALPHA for RGBA 4:4:4:4), and the samples -- sync loop and
encoder pool -- are byte-identical to the reference's."""
import json

import pytest

from test_sdk_integration_gpu import needs_build, run, shim_stats

pytestmark = pytest.mark.gpu


@needs_build
@pytest.mark.parametrize("fmt,channels", [("b64a", 3), ("b64a_rgba", 4), ("rg64", 3), ("rg64_rgba", 4)])
def test_rgba64_sources_match_reference(fmt, channels):
    w, h = 1920, 1080
    gpu = run("sdk_roundtrip", w, h, 3, 2, 24, 0, fmt)
    ref = run("sdk_roundtrip_ref", w, h, 3, 2, 24, 0, fmt)
    g, r = json.loads(gpu.stdout.strip().splitlines()[-1]), json.loads(ref.stdout.strip().splitlines()[-1])
    assert g["format"] == fmt
    assert g["sample_bytes"] == r["sample_bytes"]
    assert g["sample_digest"] == r["sample_digest"] and g["pool_sample_digest"] == r["pool_sample_digest"]
    st = shim_stats(gpu.stderr)
    assert st["fwd_gpu"] >= 4 + 32 and st["fwd_ref"] == 0 and st["cuda_errors"] == 0
    # 9 highpass bands per channel, every frame coded from the sparse format
    assert st["sparse_bands"] == 9 * channels * st["fwd_gpu"] and st["dense_bands"] == 0
