"""Weight repacking (refvsr_b200/packing.py): the SIMT matrix and the swizzled tensor-core image decode back to
the original convolution weights under the layouts documented in include/refvsr_b200.h / conv_tc.cu."""
import pytest
import torch

from refvsr_b200 import packing


def unswizzle_tc(wp, srcs, cout, kh, kw, nb):
    """inverse of pack_tc following the kernel's addressing: stage s = kx*nchunks + chunk; row r of a
    [NB][64] slab holds 16-byte chunk j at position j ^ (r % 8)."""
    nblk, S, _, _, _ = wp.shape
    allocs = [a for _, a in srcs]
    nch = [(a + 63) // 64 for a in allocs]
    nchunks = sum(nch)
    w = torch.zeros(cout, sum(allocs), kh, kw)
    t = wp.float().view(nblk, S, kh, nb, 8, 8)
    for b in range(nblk):
        for s in range(S):
            kx, ch = divmod(s, nchunks)
            src, cj = (0, ch) if ch < nch[0] else (1, ch - nch[0])
            base = (0 if src == 0 else allocs[0]) + 64 * cj
            for r in range(nb):
                n = b * nb + r
                if n >= cout:
                    continue
                row = torch.stack([t[b, s, :, r, j ^ (r % 8), :] for j in range(8)], 1).reshape(kh, 64)
                width = min(64, allocs[src] - 64 * cj)
                w[n, base:base + width, :, kx] = row[:, :width].t()
    return w


@pytest.mark.parametrize('srcs,cout,k', [([(48, 48)], 48, 3), ([(3, 8), (48, 48)], 48, 3), ([(64, 64)], 32, 7),
                                         ([(48, 48)], 192, 3), ([(16, 16)], 2, 7), ([(48, 48), (48, 48)], 48, 1),
                                         ([(96, 96)], 24, 3)])
def test_pack_tc_roundtrip(srcs, cout, k):
    cin = sum(r for r, _ in srcs)
    w = torch.randn(cout, cin, k, k).half().float()
    nb = packing.choose_nb(cout)
    assert nb % 16 == 0 and 16 <= nb <= 256
    wp = packing.pack_tc(w, srcs, torch.float16, nb)
    nchunks = sum((a + 63) // 64 for _, a in srcs)
    assert wp.shape == ((cout + nb - 1) // nb, k * nchunks, k, nb, 64)
    back = unswizzle_tc(wp, srcs, cout, k, k, nb)
    exp = packing._expand_inputs(w, srcs)
    assert torch.equal(back, exp)


def test_pack_simt_layout():
    srcs = [(3, 8), (5, 8)]
    w = torch.randn(6, 8, 3, 3)
    m = packing.pack_simt(w, srcs)
    assert m.shape == (3 * 3 * 16, 8)
    ct = 16
    for (n, c_real, c_alloc, ky, kx) in [(0, 0, 0, 0, 0), (5, 2, 2, 1, 2), (3, 4, 9, 2, 1), (2, 7, 12, 0, 1)]:
        assert m[(ky * 3 + kx) * ct + c_alloc, n] == w[n, c_real, ky, kx]
    assert m[(0 * 3 + 0) * ct + 5, 0] == 0 and m[:, 6:].abs().sum() == 0     # padding channels / columns


def test_pack_conv_chooses_impl():
    w, b = torch.randn(48, 48, 3, 3), torch.zeros(48)
    from refvsr_b200.lib import IMPL_SIMT, IMPL_TC
    assert packing.pack_conv('a', w, b, [(48, 48)], 1, 1, torch.float16, 'cpu', True).impl == IMPL_TC
    assert packing.pack_conv('a', w, b, [(48, 48)], 2, 1, torch.float16, 'cpu', True).impl == IMPL_SIMT
    assert packing.pack_conv('a', w, b, [(48, 48)], 1, 1, torch.float32, 'cpu', True).impl == IMPL_SIMT
    assert packing.pack_conv('a', w, b, [(48, 48)], 1, 1, torch.float16, 'cpu', False).impl == IMPL_SIMT
    p = packing.pack_conv('a', w, b, [(48, 48)], 1, 1, torch.float16, 'cpu', True, bias_add=1.0)
    assert torch.equal(p.bias, torch.ones(48))


@pytest.mark.parametrize('k,srcs', [(3, [(48, 48)]), (5, [(32, 32), (32, 32)]), (5, [(3, 8)])])
def test_space_to_depth_reindexing_equals_stride2_conv(k, srcs, oracle_ops):
    """stride-2 conv == stride-1 3x3 conv over the space-to-depth input with packing.s2d_weights"""
    import torch.nn.functional as F
    cin = sum(r for r, _ in srcs)
    w, b = torch.randn(7, cin, k, k), torch.randn(7)
    xs = [torch.randn(12, 18, a) for _, a in srcs]
    xin = torch.cat([x[..., :r].permute(2, 0, 1) for x, (r, _) in zip(xs, srcs)], 0).unsqueeze(0)
    exp = F.conv2d(xin, w, b, stride=2, padding=k // 2)[0].permute(1, 2, 0)
    w2, srcs2 = packing.s2d_weights(w, srcs, k // 2)
    zs = []
    for x in xs:
        z = torch.empty(6, 9, 4 * x.shape[2])
        oracle_ops.space_to_depth2(x, z)
        zs.append(z)
    layer = oracle_ops.pack_conv('s2d', w2, b, srcs2, 1, 1, torch.float32, 'cpu', False)
    out = torch.zeros(6, 9, 7)
    oracle_ops.conv2d(layer, zs[0], zs[1] if len(zs) > 1 else None, out)
    assert (out - exp).abs().max() < 1e-4


def test_layout1_image_is_tap_major_and_layout3_is_the_same_image():
    """layout 1 = [nblk][chunk][ky][kx][NB][64]: the three kx taps of one ky are ADJACENT row blocks, which is what the
    kx-folded conv mode multiplies as one N = 3 * NB operand (conv_tc.cu MODE 3); layout 3 is the same image with the
    folding disabled."""
    cout, cin, k, nb = 48, 48, 3, 48
    w = torch.randn(cout, cin, k, k).half().float()
    p1 = packing.pack_tc(w, [(cin, cin)], torch.float16, nb, layout=1)
    p3 = packing.pack_tc(w, [(cin, cin)], torch.float16, nb, layout=3)
    assert torch.equal(p1, p3)
    assert tuple(p1.shape) == (1, 1, k * k, nb, 64)
    t = p1.float().view(k * k, nb, 8, 8)
    for ky in range(k):
        for kx in range(k):
            for n in (0, 7, 13, 47):
                row = torch.stack([t[ky * k + kx, n, j ^ (n % 8)] for j in range(8)]).reshape(64)
                assert torch.equal(row[:cin], w[n, :, ky, kx]), (ky, kx, n)


def test_choose_layout_defaults_and_env(monkeypatch):
    monkeypatch.delenv('REFVSR_TC_LAYOUT', raising=False)
    assert packing.choose_layout(3, 3, [(48, 48)], 48) == 1                      # taps resident -> one box per tile
    assert packing.choose_layout(7, 7, [(64, 64)], 64) == 0                      # 49 taps x 64 x 128 B do not fit
    assert packing.choose_layout(3, 5, [(48, 48)], 48) == 0                      # non-square kernels: layout 0
    monkeypatch.setenv('REFVSR_TC_LAYOUT', '3')
    assert packing.choose_layout(3, 3, [(48, 48)], 48) == 3
    assert packing.choose_layout(7, 7, [(64, 64)], 64) == 0
    monkeypatch.setenv('REFVSR_TC_LAYOUT', '0')
    assert packing.choose_layout(3, 3, [(48, 48)], 48) == 0
