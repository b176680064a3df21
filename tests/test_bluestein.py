"""Runs the Bluestein pass's per-line steps on the CPU (tests/emu_bluestein.cpp: fft_core.cuh's stage arithmetic and the
host tables of bluestein.hpp) against a naive long-double DFT — every length 3..300 and 1000, 2047, 2049, 3000, 4093,
4095, both directions, f64 and f32, at the project tolerances."""
import os
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))


def test_bluestein_matches_naive_dft():
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "emu")
        subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(HERE, "emu_bluestein.cpp")], check=True)
        r = subprocess.run([exe], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout[-2000:]
        assert "fails=0" in r.stdout
