"""The TMA-store epilogue of conv_igemm_kernel (same-grid bf16 outputs: training forward z, every dgrad, eval stride-1
blocks): the output map clips the stores to `store_cols` channels and `np` rows, so channels beyond the view, the halo
and the neighbours in a wider (concat) buffer must come out exactly as the layout requires.  Every case is compared with
F.conv2d at the tolerances of test_conv_gpu.py, and every byte outside the view's interior is checked."""
import pytest

from builders import tma_epilogue_run

pytestmark = pytest.mark.gpu

@pytest.mark.parametrize("cfg", [
    # dgrad accumulating into a channel-offset view of a wider concat gradient buffer, halo garbage zeroed
    dict(batch=2, h=19, w=19, cin=128, cout=96, k=3, width=256, off=32, acc=True),
    dict(batch=2, h=38, w=38, cin=128, cout=256, k=1, width=768, off=256, acc=True),
    # np = 8 * 47 * 47 = 17672 = 138 * 128 + 8: partial last tile, 278 tiles (several per persistent CTA) + shortcut
    dict(batch=8, h=45, w=45, cin=64, cout=512, k=3, width=512, res_sep=True),
    # store_cols < BN in a wider buffer: 160 of 256 (the fourth 64-filter box lies wholly beyond), 96 of 128
    dict(batch=2, h=20, w=16, cin=64, cout=160, k=3, width=320),
    dict(batch=3, h=13, w=11, cin=192, cout=96, k=1, width=224),
])
def test_tma_store_epilogue_vs_torch(cfg):
    r = tma_epilogue_run(**cfg)
    assert r["within"] and r["halo_zero"] and r["pad_zero"] and r["sentinels"], r
