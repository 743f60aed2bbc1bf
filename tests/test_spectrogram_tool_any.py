"""bin/sdr_spectrogram -a (any width up to 65536, through xlg_add_spectrum_any): its refusals and help, which come
before any GPU work.  The images themselves are checked on the GPU (tests/test_gpu_spectrum_czt.py)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "sdr-server_b200", "bin", "sdr_spectrogram")


def tool(*args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")  # a refusal must come before any GPU work
    return subprocess.run([TOOL, *map(str, args)], capture_output=True, text=True, env=env, timeout=60)


@pytest.fixture
def inp(tmp_path):
    p = tmp_path / "in.cu8"
    p.write_bytes(bytes(2 * 1000))
    return p


REFUSALS = [
    (["-a", "-w", "131072", "-s", "1e6"], "-w (131072) is not served: widths up to 65536"),
    (["-a", "-w", "65537", "-s", "1e6"], "-w (65537) is not served: widths up to 65536"),
    (["-a", "-w", "5000", "-s", "4999"], "-w (5000) is too wide for sampling rate 4999"),
    (["-a", "-w", "0"], "-w (width) should be positive. got: 0"),
    (["-a", "-w", "5000", "-s", "100000", "-d", "cs8"], "unsupported data format: cs8"),
    (["-a", "-w", "5000", "-s", "100000"], "fewer than one row of 100000"),
    (["-w", "5000", "-s", "100000"], "-w (5000) is not served: widths up to 4096, or powers of two up to 65536"),
]


@pytest.mark.parametrize("args,message", REFUSALS, ids=[" ".join(a) for a, _ in REFUSALS])
def test_any_width_refusals(tmp_path, inp, args, message):
    r = tool("-i", inp, "-o", tmp_path / "out.png", *args)
    assert r.returncode != 0
    assert message in r.stderr, r.stderr
    assert not (tmp_path / "out.png").exists()


def test_help_lists_any_width():
    r = tool("-h")
    assert r.returncode == 0
    assert "-a  any width up to 65536" in r.stdout
