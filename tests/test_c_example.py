"""examples/roundtrip.c drives the library from plain C (gcc, no Python in the loop).  Without a GPU it must fail loudly
with CFB_ERROR_NO_DEVICE (there is no CPU fallback); on an H100 it must round-trip a frame, progressive and interlaced."""
import importlib
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _exe():
    import __graft_entry__ as g
    g.build_product()
    return g.build_examples()


def test_c_example_fails_loudly_without_gpu():
    pkg = importlib.import_module("cineform-sdk_b200")
    if pkg.device_count() > 0:
        pytest.skip("a GPU is present")
    p = subprocess.run([_exe(), "256", "64"], capture_output=True, text=True, timeout=120)
    assert p.returncode == 3
    assert "no CPU fallback" in p.stderr and "failed: 100" in p.stderr


@pytest.mark.parametrize("size", [("704", "96"), ("1920", "1080")])
def test_c_entropy_handover_round_trip(size):
    """examples/entropy_handover.c: sparse buffer -> band streams (cfb_sparse_vlc_band) -> sparse buffer (cfb_vlc_decode_band +
    sparse writer) from plain C with a caller-supplied code set; host only, so it runs here."""
    exe = os.path.join(os.path.dirname(_exe()), "entropy_handover")
    p = subprocess.run([exe, *size], capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stderr[-1000:]
    r = json.loads(p.stdout.strip().splitlines()[-1])
    assert r["sparse_round_trip_identical"] == 1 and r["dense_round_trip_identical"] == 1
    assert 0 < r["sparse_bytes"] < r["coded_bytes"] // 4 and r["nonzero_coefficients"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("args", [("1920", "1080", "0"), ("720", "480", "1"), ("3840", "2160", "0")])
def test_c_example_roundtrip(args):
    p = subprocess.run([_exe(), *args], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-1000:]
    r = json.loads(p.stdout.strip().splitlines()[-1])
    assert r["luma_psnr_db"] > 40.0 and r["kernel_launches"] >= 6
    assert 0 < r["nonzero_coefficients"] < r["coded_bytes"] // 2
