"""Test oracle: MobileCLIP's text student with batch-statistics BatchNorm in the RepMixerBlocks (nn.BatchNorm2d in train mode,
mobile_clip.py:545-702 under .train()).  Restates oracle.text's RepMixerBlock with F.batch_norm(training=True) on clones of the
running buffers, which the forward updates and returns; every other piece is oracle.text's.  Pure PyTorch, CPU or CUDA."""
from __future__ import annotations

import torch.nn.functional as F

from oracle import text as OT

BN_SUFFIXES = ("token_mixer.mixer.rbr_skip", "token_mixer.mixer.rbr_conv.0.bn", "token_mixer.norm.rbr_skip", "convffn.conv.bn")


def running_clones(sd):
    """{BN prefix: [running_mean, running_var, num_batches_tracked]} cloned from a state dict (detached, fp32/int64 as stored)."""
    out = {}
    for k, v in sd.items():
        if k.endswith(".running_mean"):
            p = k[: -len(".running_mean")]
            nbt = sd.get(p + ".num_batches_tracked")
            out[p] = [v.detach().clone(), sd[p + ".running_var"].detach().clone(), int(nbt) if nbt is not None else 0]
    return out


def _bn_train(x, sd, p, run, momentum=0.1, eps=1e-5):
    r = run[p]
    y = F.batch_norm(x, r[0], r[1], sd[p + ".weight"], sd[p + ".bias"], True, momentum, eps)
    r[2] += 1
    return y


def repmixer_block_bn(x, sd, p, run):
    """oracle.text.repmixer_block with every BatchNorm in train mode: x [B, L, C] -> [B, L, C]; run updated in place."""
    t = x.permute(0, 2, 1).unsqueeze(2)
    tm = p + ".token_mixer"
    # nn.Module call order of the reference: mixer (rbr_skip, then rbr_conv) before norm (mobile_clip.py:594-603)
    ms = _bn_train(t, sd, tm + ".mixer.rbr_skip", run)
    mc = _bn_train(OT._dw(t, sd[tm + ".mixer.rbr_conv.0.conv.weight"]), sd, tm + ".mixer.rbr_conv.0.bn", run)
    ns = _bn_train(t, sd, tm + ".norm.rbr_skip", run)
    t = t + sd[tm + ".layer_scale"] * (ms + mc - ns)
    f = p + ".convffn"
    u = _bn_train(OT._dw(t, sd[f + ".conv.conv.weight"]), sd, f + ".conv.bn", run)
    u = F.conv2d(F.gelu(F.conv2d(u, sd[f + ".fc1.weight"], sd[f + ".fc1.bias"])), sd[f + ".fc2.weight"], sd[f + ".fc2.bias"])
    t = t + sd[p + ".layer_scale"] * u
    return t.squeeze(2).permute(0, 2, 1)


def mobileclip_encode_bn(sd, x, cfg, run, prefix="encoder."):
    """oracle.text.mobileclip_encode with batch-statistics RepMixerBlocks."""
    mask = OT.causal_mask(x.shape[1], x.device) if cfg["causal_masking"] else None
    n = cfg["n_transformer_layers"] + (2 if cfg["model_name"] == "mct" else 0)
    for i in range(n):
        p = f"{prefix}transformer.{i}"
        if p + ".token_mixer.layer_scale" in sd:
            x = repmixer_block_bn(x, sd, p, run)
        else:
            x = OT.transformer_encoder(x, sd, p, cfg["n_heads_per_layer"], mask)
    return OT._ln(x, sd, prefix + "final_layer_norm")


def text_student_bn(sd, ids, cfg, run):
    """oracle.text.text_student in train mode: (mask, memory [L,B,out], input_embeds [L,B,dim]); run updated in place."""
    emb = OT.mobileclip_embed(sd, ids)
    mem = OT._lin(mobileclip_encode_bn(sd, emb, cfg, run), sd, "projector")
    return (ids != 0).ne(True), mem.transpose(0, 1), emb.transpose(0, 1)
