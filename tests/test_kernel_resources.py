"""Register budget of the tensor-core MLP kernels (mlp_tc.cu), read from ptxas's resource report for sm_90a.

At 512 threads and one CTA per SM a thread has at most 128 registers.  The forward kernels must fit without local-memory
spills or a stack frame, at both padded obs widths; the training kernels keep their remaining spills under a fixed bound
(2.3 KB per thread before the kernels were templated on the padded obs width).  No wgmma may be serialised by the compiler."""
import os
import re
import shutil
import subprocess

import pytest

from tianshou_b200.csrc import build as B

MLP_TC = os.path.join(B.HERE, "mlp_tc.cu")
SPILL_BOUND = 512   # bytes of spill stores / loads of ppo_tc_kernel<EPOCH, KXP>


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    if shutil.which(B.NVCC) is None and not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("ptxas") / "mlp_tc.o"
    r = subprocess.run([B.NVCC, *B.FLAGS, "-c", MLP_TC, "-o", str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    kernels = {}
    for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'\n(?:.*\n)*?\s*(\d+) bytes stack frame, (\d+) bytes spill "
                         r"stores, (\d+) bytes spill loads", log):
        kernels[m.group(1)] = (int(m.group(2)), int(m.group(3)), int(m.group(4)))
    return log, kernels


def _entry(kernels, pattern):
    hits = {k: v for k, v in kernels.items() if re.search(pattern, k)}
    assert len(hits) == 1, (pattern, sorted(kernels))
    return next(iter(hits.values()))


@pytest.mark.parametrize("kxp", [16, 32])
@pytest.mark.parametrize("kernel", ["forward_tc_kernelILi0ELi{}E", "forward_tc_kernelILi1ELi{}E"])
def test_spill_free(report, kernel, kxp):
    stack, spill_st, spill_ld = _entry(report[1], kernel.format(kxp))
    assert (stack, spill_st, spill_ld) == (0, 0, 0)


@pytest.mark.parametrize("kxp", [16, 32])
@pytest.mark.parametrize("epoch", [0, 1])
def test_training_kernel_spill_bound(report, epoch, kxp):
    stack, spill_st, spill_ld = _entry(report[1], f"ppo_tc_kernelILb{epoch}ELi{kxp}E")
    assert spill_st <= SPILL_BOUND and spill_ld <= SPILL_BOUND, (stack, spill_st, spill_ld)


def test_no_serialized_wgmma(report):
    assert "serialized" not in report[0]
