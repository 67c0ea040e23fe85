"""Auxiliary losses through the fast encoders (x_clip_b200/aux.py, SURVEY 8f rank 4): multiview
against the reference's golden values, MLM and SimSiam/SimCLR against fp32 restatements built on the
oracle encoders with the random parts pinned (a fixed corruption, identity augmentation)."""
import json
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"
TINY = dict(dim_text=256, dim_image=256, dim_latent=256, num_text_tokens=128, text_enc_depth=2,
            text_seq_len=16, text_heads=4, visual_enc_depth=2, visual_heads=4,
            visual_image_size=64, visual_patch_size=16)


@pytest.mark.parametrize("case", ["tiny_multiview", "tiny_multiview_dcl_extra"])
def test_multiview_matches_reference(cuda_device, case):
    from oracle import clip_oracle as O
    import x_clip_b200
    gold = json.loads((GOLD / f"{case}.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    nv = 1 + max(gold["n_aug_text"], gold["n_aug_image"])
    views = [O.protocol_inputs(cfg, gold["batch"], gold["input_seed"] + gold["view_seed_stride"] * v,
                               gold["pad_fraction"]) for v in range(nv)]
    texts = [views[v][0].to(cuda_device) for v in range(1 + gold["n_aug_text"])]
    images = [views[v][1].to(cuda_device) for v in range(1 + gold["n_aug_image"])]
    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0.).to(cuda_device)
    clip.load_state_dict(state)
    clip.train()
    loss = clip(texts[0], images[0], return_loss=True,
                aug_text=tuple(texts[1:]) if gold["n_aug_text"] else None,
                aug_image=tuple(images[1:]) if gold["n_aug_image"] else None)
    loss.backward()
    assert abs(loss.item() - gold["loss"]) <= 1e-3 * abs(gold["loss"])
    gn = torch.sqrt(sum((p.grad.double() ** 2).sum() for p in clip.parameters() if p.grad is not None)).item()
    assert abs(gn - gold["grad_norm"]) <= 1e-2 * gold["grad_norm"], (gn, gold["grad_norm"])
    assert abs(clip.temperature.grad.item() - gold["dtemperature"]) <= 1e-2 * abs(gold["dtemperature"]) + 1e-3


def test_mlm_loss_matches_fp32_restatement(cuda_device):
    """reference mlm.py:69-107 with the corruption pinned: encode the corrupted sequence, project
    the chosen positions onto the vocabulary, cross entropy against the original tokens."""
    from oracle import clip_oracle as O
    import x_clip_b200
    kw = dict(TINY, num_text_tokens=120)             # + [MASK] -> 121 rows in the embedding table; the
    # 120-way vocabulary projection of the masked rows runs on the wgmma GEMM (N % 8 == 0)
    clip = x_clip_b200.CLIP(**kw, use_mlm=True, mlm_mask_token_id=2, visual_patch_dropout=0.).to(cuda_device)
    clip.train()
    cfg = O.ClipConfig(**dict(kw, num_text_tokens=121))
    text, _ = O.protocol_inputs(cfg, 6, 11, 0.2)
    text = text.clamp(max=119).to(cuda_device)
    torch.manual_seed(3)
    masked, labels = clip.mlm.corrupt(text)
    sel = labels != 0
    assert sel.any() and (labels[sel] == text[sel]).all() and (masked[~sel] == text[~sel]).all()
    assert sel.sum(dim=-1).max().item() <= -(-16 * 15 // 100) + 1          # ~ceil(0.15 * maskable) per row
    loss = clip.mlm.loss_from(masked, labels, mask=text != 0)
    loss.backward()
    p = {k: v.detach().float().cpu() for k, v in clip.state_dict().items() if not k.startswith("mlm.")}
    enc = O.encode_text(masked.cpu(), (text != 0).cpu(), p, cfg)[:, 1:]
    logits = F.linear(enc[sel.cpu()], clip.mlm.to_logits.weight.detach().cpu(), clip.mlm.to_logits.bias.detach().cpu())
    ref = F.cross_entropy(logits, labels.cpu()[sel.cpu()])
    assert abs(loss.item() - ref.item()) <= 5e-3 * abs(ref.item()), (loss.item(), ref.item())
    assert clip.mlm.to_logits.weight.grad.abs().sum() > 0
    assert clip.text_transformer.token_emb.weight.grad.abs().sum() > 0

    # and inside CLIP.forward the weights are the reference's (:858-865)
    torch.manual_seed(5)
    total = clip(text, torch.randn(6, 3, 64, 64, device=cuda_device), return_loss=True)
    assert torch.isfinite(total)


@pytest.mark.parametrize("kind", ["simsiam", "simclr"])
def test_visual_ssl_with_identity_augmentation(cuda_device, kind):
    from oracle import clip_oracle as O
    import x_clip_b200
    from x_clip_b200 import aux
    clip = x_clip_b200.CLIP(**TINY, visual_patch_dropout=0.).to(cuda_device)
    net = clip.visual_transformer
    ident = torch.nn.Identity()
    torch.manual_seed(0)
    if kind == "simsiam":
        ssl = aux.SimSiam(net, image_size=64, rep_dim=256, projection_hidden_size=64, augment_fn=ident).to(cuda_device)
    else:
        ssl = aux.SimCLR(net, image_size=64, rep_dim=256, project_dim=32, augment_fn=ident).to(cuda_device)
    ssl.train()
    img = torch.randn(5, 3, 64, 64, device=cuda_device)
    loss = ssl(img)
    loss.backward()
    assert torch.isfinite(loss) and net.to_tokens[1].weight.grad.abs().sum() > 0
    # fp32 restatement on the oracle's vision encoder with the same head weights
    cfg = O.ClipConfig(**TINY)
    p = {k: v.detach().float().cpu() for k, v in clip.state_dict().items()}
    rep = O.encode_image(img.cpu(), p, cfg)[:, 0]
    import copy
    if kind == "simsiam":
        proj = copy.deepcopy(ssl.online_encoder.projector).cpu().train()
        pred = copy.deepcopy(ssl.online_predictor).cpu().train()
        z = proj(rep)
        q = pred(z)
        ref = (2 * (2 - 2 * (F.normalize(q, dim=-1) * F.normalize(z.detach(), dim=-1)).sum(-1))).mean()
    else:
        proj = copy.deepcopy(ssl.net.projector).cpu().train()
        z = torch.cat((proj(rep), proj(rep)))
        lg = (z @ z.t() / 0.1).masked_fill(torch.eye(10, dtype=torch.bool), -torch.finfo(torch.float32).max)
        ref = F.cross_entropy(lg, torch.cat((torch.arange(5, 10), torch.arange(0, 5))))
    assert abs(loss.item() - ref.item()) <= 2e-2 * abs(ref.item()) + 2e-3, (loss.item(), ref.item())
