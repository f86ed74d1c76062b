"""Host-side pieces of the GroundingDINO acceleration layer that need no GPU: which HF modules ``accelerate`` replaces, and that
it leaves transformers' modelling code as it found it."""
import torch

from vlfm_b200.vlm import gdino_accel as ga


def test_accelerate_replaces_every_layer_class_and_patches_nothing():
    from transformers import GroundingDinoConfig, GroundingDinoForObjectDetection
    from transformers.models.grounding_dino import modeling_grounding_dino as mgd

    cfg = GroundingDinoConfig()
    cfg.encoder_layers = cfg.decoder_layers = 2
    m = GroundingDinoForObjectDetection(cfg)
    info = ga.accelerate(m)
    assert info["deformable_layers"] == 2 and info["fusion_layers"] == 2 and info["decoder_layers"] == 2 and info["linear"] > 20
    replaced = (mgd.GroundingDinoDecoderLayer, mgd.GroundingDinoDeformableLayer, mgd.GroundingDinoFusionLayer,
                mgd.MultiScaleDeformableAttention, mgd.GroundingDinoMultiscaleDeformableAttention)
    left = [type(x).__name__ for x in m.modules() if isinstance(x, replaced)]
    assert not left, left
    assert mgd.torch is torch                      # no process-wide patch of the modelling module
