"""Register budget of the tensor-core MLP kernels (mlp_tc.cu), read from ptxas's resource report for sm_90a.

At 512 threads and one CTA per SM a thread has at most 128 registers.  The forward kernels must fit without local-memory
spills or a stack frame, at both padded obs widths; the training kernels keep their remaining spills under a fixed bound
(2.3 KB per thread before the kernels were templated on the padded obs width).  No wgmma may be serialised by the compiler."""
import os
import re

import pytest

from offpolicy_testutil import parse_ptxas, ptxas_log
from tianshou_b200.csrc import build as B

MLP_TC = os.path.join(B.HERE, "mlp_tc.cu")
SPILL_BOUND = 512   # bytes of spill stores / loads of ppo_tc_kernel<EPOCH, KXP>


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    log = ptxas_log(MLP_TC, tmp_path_factory.mktemp("ptxas"))
    return log, parse_ptxas(log)


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
