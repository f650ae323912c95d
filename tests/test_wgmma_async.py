"""SASS-level guard: the convolution wgmma kernels keep their MMAs asynchronous.  When ptxas serializes wgmmas (C7511) every
HGMMA is followed by a full drain (WARPGROUP.DEPBAR.LE gsb0, 0x0); a slab kernel that waits once per k-tile drains after
every 4 HGMMAs.  The weight-gradient kernels retire k-tiles one behind (DEPBAR.LE gsb0, 0x1) and drain once, the slab
kernels drain once per tile."""
import functools
import subprocess

import pytest

from deeprl_b200 import _lib


@functools.lru_cache(maxsize=1)
def _conv_kernel_counts():
    """{convolution kernel: [HGMMA, WARPGROUP.DEPBAR, DEPBAR.LE gsb0 0x0, DEPBAR.LE gsb0 0x1]} from the library's SASS."""
    import shutil
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    counts = {}
    name = None
    for line in sass.splitlines():
        if "Function :" in line:
            name = line.split("Function :")[1].strip()
            counts[name] = [0, 0, 0, 0]
        elif name is not None:
            counts[name][0] += "HGMMA" in line
            counts[name][1] += "WARPGROUP.DEPBAR" in line
            counts[name][2] += "WARPGROUP.DEPBAR.LE gsb0, 0x0" in line
            counts[name][3] += "WARPGROUP.DEPBAR.LE gsb0, 0x1" in line
    return {k: v for k, v in counts.items() if "conv_wgrad_wgmma_kernel" in k or "conv_slab_wgmma_kernel" in k}


def test_conv_wgmma_kernels_do_not_drain_per_ktile():
    conv = _conv_kernel_counts()
    assert sum("conv_wgrad" in k for k in conv) >= 4 and sum("conv_slab" in k for k in conv) >= 9, sorted(conv)
    for k, (mma, waits, drains, _) in conv.items():
        assert mma >= 12, (k, mma)
        assert drains <= mma // 8, "%s: %d full drains for %d HGMMA" % (k, drains, mma)
        assert waits <= mma // 4 + 1, "%s: %d waits for %d HGMMA" % (k, waits, mma)


def test_wgrad_kernels_retire_a_ktile_before_releasing_its_stage():
    """The weight-gradient kernels release k-tile i - 1's shared-memory stage only after wgmma.wait_group 1 has retired it.
    Without that wait the stage can be refilled while its MMAs still read it -- a race that rarely changes a value, so no
    numerical test catches its loss reliably: the wait itself is checked here."""
    wgrad = {k: v for k, v in _conv_kernel_counts().items() if "conv_wgrad" in k}
    assert len(wgrad) >= 4, sorted(wgrad)
    for k, (_, _, _, retire_one) in wgrad.items():
        assert retire_one >= 1, "%s: no WARPGROUP.DEPBAR.LE gsb0, 0x1 (wgmma.wait_group 1)" % k
