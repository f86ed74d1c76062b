"""The mobile_sam checkpoint names map onto the engine layout: exact key set and shapes, dropped keys, unknown keys raise."""
import pytest
import torch

from vlfm_b200.vlm.sam_config import TINY, VIT_T, SamDims, random_state_dict
from vlfm_b200.vlm.sam_weights import convert_state_dict


def expected_shapes(d: SamDims):
    E, P = d.embed_dims, d.prompt_dim
    pad8 = lambda k: (k + 7) // 8 * 8
    s = {"stem0.w": (d.stem_mid, 32), "stem0.b": (d.stem_mid,), "stem1.w": (E[0], pad8(9 * d.stem_mid)), "stem1.b": (E[0],)}
    for st in range(len(E)):
        C = E[st]
        for b in range(d.depths[st]):
            p = f"l{st}.b{b}."
            if st == 0:
                hid = C * d.mbconv_ratio
                s.update({p + "conv1.w": (hid, C), p + "conv1.b": (hid,), p + "conv2.w": (9, hid), p + "conv2.b": (hid,),
                          p + "conv3.w": (C, hid), p + "conv3.b": (C,)})
                continue
            ws = d.windows[st]
            s.update({p + "ln1.w": (C,), p + "ln1.b": (C,), p + "qkv.w": (3 * C, C), p + "qkv.b": (3 * C,),
                      p + "bias": (d.heads[st], ws * ws), p + "proj.w": (C, C), p + "proj.b": (C,), p + "local.w": (9, C),
                      p + "local.b": (C,), p + "ln2.w": (C,), p + "ln2.b": (C,), p + "fc1.w": (4 * C, C), p + "fc1.b": (4 * C,),
                      p + "fc2.w": (C, 4 * C), p + "fc2.b": (C,)})
        if st + 1 < len(E):
            Co = E[st + 1]
            p = f"l{st}.down."
            s.update({p + "conv1.w": (Co, C), p + "conv1.b": (Co,), p + "conv2.w": (9, Co), p + "conv2.b": (Co,),
                      p + "conv3.w": (Co, Co), p + "conv3.b": (Co,)})
    s.update({"neck0.w": (P, E[-1]), "neck1.w": (P,), "neck1.b": (P,), "neck2.w": (P, 9 * P), "neck3.w": (P,), "neck3.b": (P,),
              "pe.gauss": (2, P // 2), "no_mask": (P,), "fixed": (7, P), "up1.w": (P, P), "up1.b": (P,), "up_ln.w": (P // 4,),
              "up_ln.b": (P // 4,), "up2.w": (P // 2, P // 4), "up2.b": (P // 2,), "hyper0.w": (P, P), "hyper0.b": (P,),
              "hyper1.w": (P, P), "hyper1.b": (P,), "hyper2.w": (P // 8, P), "hyper2.b": (P // 8,),
              "norm_final.w": (P,), "norm_final.b": (P,)})

    def attn(p, inner):
        for a in "qkv":
            s.update({f"{p}.{a}.w": (inner, P), f"{p}.{a}.b": (inner,)})
        s.update({f"{p}.o.w": (P, inner), f"{p}.o.b": (P,)})

    for i in range(d.dec_depth):
        p = f"dec{i}"
        attn(p + ".self", P)
        attn(p + ".t2i", P // 2)
        attn(p + ".i2t", P // 2)
        for n in range(1, 5):
            s.update({f"{p}.norm{n}.w": (P,), f"{p}.norm{n}.b": (P,)})
        s.update({p + ".mlp1.w": (d.dec_mlp, P), p + ".mlp1.b": (d.dec_mlp,), p + ".mlp2.w": (P, d.dec_mlp), p + ".mlp2.b": (P,)})
    attn("final", P // 2)
    return s


@pytest.mark.parametrize("d", [VIT_T, TINY], ids=["vit_t", "tiny"])
def test_converted_keys_and_shapes(d):
    sd = random_state_dict(d, 0)
    assert any(k.startswith("image_encoder.head.") for k in sd) and any(k.startswith("image_encoder.norm_head.") for k in sd)
    out = convert_state_dict(sd, d)
    exp = expected_shapes(d)
    assert sorted(out) == sorted(exp)
    for k, shape in exp.items():
        assert tuple(out[k].shape) == shape, k
        assert out[k].dtype == torch.float32


def test_qkv_rows_permuted_per_head():
    d = TINY
    sd = random_state_dict(d, 0)
    out = convert_state_dict(sd, d)
    C, H = d.embed_dims[1], d.heads[1]
    hd = C // H
    w = sd["image_encoder.layers.1.blocks.0.attn.qkv.weight"]
    for h in range(H):
        for j, name in enumerate("qkv"):
            assert torch.equal(out["l1.b0.qkv.w"][j * C + h * hd:j * C + (h + 1) * hd], w[h * 3 * hd + j * hd:h * 3 * hd + (j + 1) * hd])


def test_dropped_and_unknown_keys():
    d = TINY
    sd = random_state_dict(d, 0)
    sd["image_encoder.layers.1.blocks.0.attn.attention_bias_idxs"] = torch.zeros(49, 49, dtype=torch.long)
    sd["pixel_mean"] = torch.zeros(3, 1, 1)
    base = convert_state_dict(sd, d)
    assert not any("head" in k and "hyper" not in k for k in base)
    bad = dict(sd)
    bad["image_encoder.layers.1.blocks.0.attn.extra"] = torch.zeros(1)
    with pytest.raises(KeyError, match="unknown"):
        convert_state_dict(bad, d)
    missing = dict(sd)
    del missing["mask_decoder.transformer.norm_final_attn.weight"]
    with pytest.raises(KeyError, match="missing"):
        convert_state_dict(missing, d)
