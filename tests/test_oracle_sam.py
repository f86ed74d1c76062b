"""CPU checks of MobileSAM's host-side pieces: the Pillow-exact bilinear tables, BatchNorm folding, and the oracle's TinyViT
window attention."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torchvision.transforms.functional import resize, to_pil_image

from oracle.sam_oracle import SamOracle, preprocess, preshape
from vlfm_b200.vlm.preprocess import bilinear_tables, resize_numpy
from vlfm_b200.vlm.sam_config import TINY, random_state_dict
from vlfm_b200.vlm.sam_weights import fold_conv_bn, offset_index


@pytest.mark.parametrize("hw", [(480, 640), (640, 480), (1024, 1024), (333, 517), (1536, 2048)])
def test_bilinear_tables_match_pillow(hw):
    rng = np.random.default_rng(hw[0] * 7 + hw[1])
    img = rng.integers(0, 256, (*hw, 3), dtype=np.uint8)
    img[: hw[0] // 3] = (img[: hw[0] // 3] // 64) * 64          # flat bands and sharp edges besides noise
    newh, neww = preshape(hw[0], hw[1], 1024)
    ref = np.array(resize(to_pil_image(img), [newh, neww]))
    assert np.array_equal(resize_numpy(img, newh, neww, tables=bilinear_tables), ref)


def test_bilinear_tables_downscale_support():
    b, kk, ksize = bilinear_tables(2048, 1024)
    assert ksize == 5 and int(b[:, 1].max()) == 4
    assert np.all(kk.sum(1) >= (1 << 22) - 4) and np.all(kk.sum(1) <= (1 << 22) + 4)


def test_oracle_preprocess_pads_with_zeros():
    img = np.full((120, 160, 3), 200, np.uint8)
    x, (newh, neww) = preprocess(img, 256)
    assert (newh, neww) == (192, 256)
    assert torch.all(x[:, :, newh:] == 0)
    assert torch.allclose(x[0, :, 0, 0], (200 - torch.tensor([123.675, 116.28, 103.53])) / torch.tensor([58.395, 57.12, 57.375]))


def test_folded_conv_bn_matches_unfolded():
    sd = random_state_dict(TINY, 3)
    for name, groups in (("image_encoder.patch_embed.seq.2", 1), ("image_encoder.layers.0.blocks.0.conv2", 128)):
        x = torch.randn(2, sd[name + ".c.weight"].shape[1] * groups, 9, 11)
        ref = F.batch_norm(F.conv2d(x, sd[name + ".c.weight"], padding=1, groups=groups), sd[name + ".bn.running_mean"],
                           sd[name + ".bn.running_var"], sd[name + ".bn.weight"], sd[name + ".bn.bias"], False, 0.0, 1e-5)
        w, b = fold_conv_bn(sd, name)
        got = F.conv2d(x, w, b, padding=1, groups=groups)
        assert (got - ref).abs().max().item() <= 1e-5 * max(1.0, ref.abs().max().item())


def test_offset_index_window7():
    idx = offset_index(7)
    assert len(idx) == 49 and sorted(idx.values()) == list(range(49))
    assert all(idx[(dy, dx)] == dy * 7 + dx for dy in range(7) for dx in range(7))


def test_window_attention_without_padding_is_per_window():
    """At a resolution that is a window multiple the padded path is not taken; the result equals attention on each window."""
    sd = random_state_dict(TINY, 1)
    orc = SamOracle(TINY, sd)
    name = "image_encoder.layers.1.blocks.0"
    C, heads, ws = TINY.embed_dims[1], TINY.heads[1], TINY.windows[1]
    x = torch.randn(1, 2 * ws, 2 * ws, C)
    got = orc.tinyvit_block(x, name, heads, ws)
    a = torch.empty_like(x)
    for wy in range(2):
        for wx in range(2):
            t = x[:, wy * ws:(wy + 1) * ws, wx * ws:(wx + 1) * ws].reshape(1, ws * ws, C)
            a[:, wy * ws:(wy + 1) * ws, wx * ws:(wx + 1) * ws] = orc.window_attention(t, name + ".attn", heads, ws).view(1, ws, ws, C)
    y = x + a
    y = orc.conv_bn(y.permute(0, 3, 1, 2), name + ".local_conv", 1, C).permute(0, 2, 3, 1)
    ref = y + orc.lin(F.gelu(orc.lin(orc.ln(y, name + ".mlp.norm"), name + ".mlp.fc1")), name + ".mlp.fc2")
    assert torch.allclose(got, ref, atol=1e-5, rtol=1e-5)
