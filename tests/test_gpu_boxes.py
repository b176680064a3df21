"""Box-distributed plans (dfft_plan_create_boxes) replayed on one GPU with the real kernels.

The step lists of every rank of a box plan run in lock step through dfft_debug_run_step (gpu_replay.py): the reshape
copies (fft_copy_kernel) move the caller's boxes into and out of the natural layouts, the FFT passes are those of the
natural plan.  Each case is checked
  1. bit for bit against the same plan with natural boxes, replayed the same way, its output re-sliced to the boxes (the
     passes are identical and the copies exact);
  2. against the long-double reference within the bounds of test_gpu_schedule_replay (rel-L2 <= 3 u sqrt(sum log2 L),
     max <= 30 times that times rms(ref));
  3. the checks gpu_replay.output makes of every plan: inputs unchanged, no output element left unwritten, and the ranks
     of a step in either order giving the same bits.
With a scale, the output equals the unscaled output times the scale, bit for bit."""
import os
import subprocess
from dataclasses import replace

import numpy as np
import pytest

import distributedfft_b200 as dfft
import test_gpu_schedule_replay as G
from gpu_replay import assemble, output, replay, same_bits
from test_boxes import CASES, S3, bricks, nzc, plan

SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
C2C, R2C, DCT = dfft.C2C, dfft.R2C, dfft.DCT
P2P, A2A = 0, 1
HERE = os.path.dirname(os.path.abspath(__file__))


def check_box_plan(p, inverse, d=3, seed=0):
    x, x_ld = G.global_input(p, inverse, d, seed)
    got = output(p, inverse, d, x)
    # 1: the natural plan, replayed the same way
    want = assemble(replay(replace(p, in_boxes=None, out_boxes=None), inverse, d, x))
    assert same_bits(got, want), f"differs from the natural plan at {np.argwhere(got != want)[:8].tolist()}"
    # 2: the long-double reference
    rel, mx = G.error_check(G.geometry(p, d), got, G.reference(p, inverse, d, x_ld))
    assert rel <= 3.0 and mx <= 30.0, (rel, mx)
    return x, got


def with_comm(case, comm):
    _, P, decomp, shape, p1, p2, transform, ib, ob = case
    return plan(P, decomp, shape, p1, p2, transform=transform, in_boxes=ib, out_boxes=ob, comm=comm)


@pytest.mark.gpu
@pytest.mark.parametrize("comm", [P2P, A2A], ids=["p2p", "a2a"])
@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_box_replay(case, inv, comm):
    check_box_plan(with_comm(case, comm), inv)


@pytest.mark.gpu
@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("decomp,p1,p2", [(SL, 1, 1), (PE, 2, 2)], ids=["slab", "pencil"])
def test_box_replay_partial(decomp, p1, p2, d, inv):
    p = plan(4, decomp, S3, p1, p2, in_boxes=bricks(S3, (2, 2, 1), uneven=True), out_boxes=bricks(S3, (1, 2, 2)))
    check_box_plan(p, inv, d)


@pytest.mark.gpu
@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
def test_box_replay_x_kept(inv):
    p = plan(4, PE, S3, 2, 2, in_boxes=bricks(S3, (2, 2, 1)), out_boxes=bricks(S3, (1, 2, 2)), axes=(0, 1, 1))
    check_box_plan(p, inv)


@pytest.mark.gpu
@pytest.mark.parametrize("comm", [P2P, A2A], ids=["p2p", "a2a"])
@pytest.mark.parametrize("transform", [C2C, R2C])
def test_box_scale_is_exact(transform, comm):
    """batch 2 with a scale: the unscaled output times the scale, bit for bit"""
    ob = bricks((8, 8, nzc(plan(1, SL, S3, transform=transform))), (2, 2, 1))
    kw = dict(transform=transform, in_boxes=bricks(S3, (2, 1, 2)), out_boxes=ob, comm=comm, batch=2)
    scale = (0.37, 1.0 / 96)
    for inv in (0, 1):
        x, plain = check_box_plan(plan(4, PE, S3, 2, 2, **kw), inv)
        scaled = output(plan(4, PE, S3, 2, 2, scale=scale, **kw), inv, 3, x)
        # each real value times s (a complex product would turn the sign of zero imaginary parts)
        r = plain.real.dtype
        want = (np.ascontiguousarray(plain).view(r) * r.type(scale[inv])).view(plain.dtype)
        assert same_bits(scaled, want)


@pytest.mark.gpu
def test_cpp_shim(tmp_path):
    """tests/cpp/boxes_shim_test.cpp: the shim's box initFFT, its getters on 4 geometry-only ranks and one rank's execs"""
    exe = str(tmp_path / "boxes_shim_test")
    root = os.path.dirname(HERE)
    libdir = os.path.join(root, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(root, "include"), "-I/usr/local/cuda/include",
                    os.path.join(HERE, "cpp", "boxes_shim_test.cpp"), "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64",
                    "-lcudart", "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout + r.stderr
