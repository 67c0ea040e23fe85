"""The MLM head's vocabulary cross-entropy fused into the wgmma GEMM (xclip_vocab_ce_fwd / _bwd,
engine.VocabCrossEntropyFn) against fp64 F.cross_entropy(F.linear(...)) on bf16-exact inputs: the
loss and the gradients of the rows, the weight and the bias.

Gates are relative errors (Frobenius for the gradients), about twice the largest error measured on
an H100 80GB HBM3 (700 W power limit) over the cases below: loss 1.8e-7, d rows 3.1e-3, d weight
2.6e-3, d bias 2.7e-3.  The loss is reduced in fp32 from fp32 logits.  The gradients go through
g = gscale (softmax - onehot) rounded to bf16, which keeps them near 2^-9.

A label outside [0, V) is a device-side assert on CUDA tensors; that ends the process's CUDA
context, so tests/test_vocab_ce_plan.py checks the same engine.check_labels on CPU tensors."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32

LOSS_GATE = 4e-7
DX_GATE = 6.5e-3
DW_GATE = 5.5e-3
DB_GATE = 5.5e-3


def _inputs(n, V, d, seed, dev, bias=True, logit_span=None):
    """bf16-exact rows and weight, fp32 bias, labels with the tile edges and both ends."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn((n, d), generator=gen, device=dev).to(BF16)
    w = (torch.randn((V, d), generator=gen, device=dev) * d ** -0.5).to(BF16).float()
    b = None
    if bias:
        b = torch.randn((V,), generator=gen, device=dev) * 0.5
        if logit_span is not None:                         # logits near +-logit_span
            b = (torch.rand((V,), generator=gen, device=dev) * 2.0 - 1.0) * logit_span
    labels = torch.randint(0, V, (n,), generator=gen, device=dev)
    edges = [c for c in (0, V - 1, 127, 128, 255, 256, 257, 511, 512) if c < V]
    labels[: min(n, len(edges))] = torch.tensor(edges[:n], device=dev)
    return x, w, b, labels


def _ref64(x, w, b, labels, upstream):
    x64 = x.double().requires_grad_(True)
    w64 = w.double().requires_grad_(True)
    b64 = None if b is None else b.double().requires_grad_(True)
    loss = F.cross_entropy(F.linear(x64, w64, b64), labels)
    (loss * upstream).backward()
    return loss.detach(), x64.grad, w64.grad, None if b64 is None else b64.grad


def _rel(a, ref):
    a, ref = a.double(), ref.double()
    den = ref.norm().item()
    num = (a - ref).norm().item()
    return num / den if den > 0 else num


def _run(x, w, b, labels, upstream, need_w=True, need_b=True):
    from x_clip_b200 import engine as E
    rows = x.clone().requires_grad_(True)
    wp = w.clone().requires_grad_(need_w)
    bp = None if b is None else b.clone().requires_grad_(need_b)
    loss = E.VocabCrossEntropyFn.apply(rows, wp, bp, labels)
    (loss * upstream).backward()
    return loss.detach(), rows.grad, wp.grad, None if bp is None else bp.grad


def _check(x, w, b, labels, upstream=0.7):
    loss, dx, dw, db = _run(x, w, b, labels, upstream)
    rloss, rdx, rdw, rdb = _ref64(x, w, b, labels, upstream)
    errs = dict(loss=abs(loss.item() - rloss.item()) / max(abs(rloss.item()), 1e-30),
                dx=_rel(dx, rdx), dw=_rel(dw, rdw))
    if b is not None:
        errs["db"] = _rel(db, rdb)
    print(f"vocab_ce n={x.shape[0]} V={w.shape[0]} d={x.shape[1]} errors {errs}")
    assert dx.dtype == BF16 and dw.dtype == F32
    assert errs["loss"] <= LOSS_GATE, errs
    assert errs["dx"] <= DX_GATE, errs
    assert errs["dw"] <= DW_GATE, errs
    if b is not None:
        assert errs["db"] <= DB_GATE, errs
    return errs


@pytest.mark.parametrize("n,V,d", [(1, 8, 128), (7, 121, 128), (300, 256, 128), (129, 257, 256),
                                   (513, 10001, 512), (1000, 10000, 512), (4099, 49408, 768)])
def test_vocab_ce_matches_fp64(cuda_device, n, V, d):
    _check(*_inputs(n, V, d, 1000 + V, cuda_device))


@pytest.mark.parametrize("n,V,d", [(64, 121, 128), (600, 10001, 256)])
def test_vocab_ce_logits_near_80(cuda_device, n, V, d):
    """Logits spread over [-80, 80]: the online maximum keeps exp from overflowing fp32."""
    x, w, b, labels = _inputs(n, V, d, 7 + V, cuda_device, logit_span=80.0)
    logits = F.linear(x.double(), w.double(), b.double())
    assert logits.max().item() > 70 and logits.min().item() < -70
    _check(x, w, b, labels)


def test_vocab_ce_single_class(cuda_device):
    """V = 1: lse equals the target logit, so the loss and every gradient vanish."""
    x, w, b, labels = _inputs(5, 1, 128, 3, cuda_device)
    loss, dx, dw, db = _run(x, w, b, labels, 1.0)
    assert abs(loss.item()) <= 1e-5
    assert max(t.abs().max().item() for t in (dx, dw, db)) <= 1e-6


def test_vocab_ce_bias_free(cuda_device):
    _check(*_inputs(333, 1000, 256, 11, cuda_device, bias=False))


@pytest.mark.parametrize("budget_rows", [50, 128])
def test_vocab_ce_windows(cuda_device, monkeypatch, budget_rows):
    """Backward windows smaller than the batch (below and at 128 rows, with a partial last window)
    give the rows' gradient bit for bit and stay inside the fp64 gates."""
    from x_clip_b200 import engine as E
    x, w, b, labels = _inputs(517, 10001, 256, 21, cuda_device)
    whole = _run(x, w, b, labels, 0.7)
    ldg = (10001 + 7) // 8 * 8
    monkeypatch.setattr(E, "VOCAB_CE_WINDOW_BYTES", 2 * ldg * budget_rows + 5)
    assert E.vocab_window_rows(517, 10001) == budget_rows
    windowed = _run(x, w, b, labels, 0.7)
    assert torch.equal(windowed[0], whole[0])
    assert torch.equal(windowed[1], whole[1])
    _check(x, w, b, labels)


def test_vocab_ce_frozen_head_does_no_weight_work(cuda_device):
    """A frozen head: the rows still get their gradient, the weight and bias none, and the backward
    launches only the g kernel and the dgrad GEMM per window."""
    from x_clip_b200 import _lib
    from x_clip_b200 import engine as E
    lib = _lib.load()
    x, w, b, labels = _inputs(400, 10001, 256, 31, cuda_device)
    ref = _run(x, w, b, labels, 0.7)

    def backward_launches(need_w, need_b):
        rows = x.clone().requires_grad_(True)
        wp, bp = w.clone().requires_grad_(need_w), b.clone().requires_grad_(need_b)
        loss = E.VocabCrossEntropyFn.apply(rows, wp, bp, labels)
        torch.cuda.synchronize()
        before = lib.xclip_launch_count()
        (loss * 0.7).backward()
        torch.cuda.synchronize()
        return lib.xclip_launch_count() - before, rows.grad, wp.grad, bp.grad

    n_all, dx_all, dw_all, db_all = backward_launches(True, True)
    n_frozen, dx_frozen, dw_frozen, db_frozen = backward_launches(False, False)
    assert dw_frozen is None and db_frozen is None
    assert dw_all is not None and db_all is not None
    assert torch.equal(dx_frozen, dx_all) and torch.equal(dx_all, ref[1])
    assert n_frozen == 2 and n_all == 4, (n_frozen, n_all)


def test_vocab_ce_refuses_bad_arguments(cuda_device):
    from x_clip_b200 import _lib
    from x_clip_b200 import kernels as K
    x, w, b, labels = _inputs(16, 100, 128, 41, cuda_device)
    wb = w.to(BF16)
    with pytest.raises(_lib.XClipB200Error):
        K.vocab_ce_fwd(x, wb, b, labels.int())                       # int32 labels
    with pytest.raises(_lib.XClipB200Error):
        K.vocab_ce_fwd(x, wb, b[:99], labels)                        # bias of the wrong length
    with pytest.raises(_lib.XClipB200Error):
        K.vocab_ce_fwd(x[:, :124].contiguous(), wb[:, :124].contiguous(), b, labels)   # d % 8 != 0
    with pytest.raises(_lib.XClipB200Error):
        K.vocab_ce_fwd(x[:0], wb, b, labels[:0])                     # no rows
    with pytest.raises(_lib.XClipB200Error):
        K.vocab_ce_bwd(x, wb, b, labels, torch.zeros(16, device=x.device), torch.ones(1, device=x.device),
                       out=torch.empty((16, 100), device=x.device, dtype=BF16))   # ldg < roundup8(V)


def test_mlm_head_any_vocabulary(cuda_device):
    """aux.MLM.loss_from at a vocabulary that is not a multiple of 8 runs the fused head: the loss and
    the head's gradients match fp64 on the encodings the text tower produced."""
    import x_clip_b200
    kw = dict(dim_text=256, dim_image=256, dim_latent=256, num_text_tokens=1001, text_enc_depth=2,
              text_seq_len=16, text_heads=4, visual_enc_depth=2, visual_heads=4,
              visual_image_size=64, visual_patch_size=16)
    clip = x_clip_b200.CLIP(**kw, use_mlm=True, mlm_mask_token_id=2, visual_patch_dropout=0.).to(cuda_device)
    clip.train()
    gen = torch.Generator(device=cuda_device).manual_seed(5)
    text = torch.randint(3, 1001, (8, 16), generator=gen, device=cuda_device)
    text[:, 12:] = 0
    torch.manual_seed(3)
    masked, labels = clip.mlm.corrupt(text)
    loss = clip.mlm.loss_from(masked, labels, mask=text != 0)
    loss.backward()
    with torch.no_grad():
        enc = clip.mlm.transformer(masked, mask=text != 0)[:, 1:]
    sel = labels != 0
    head = clip.mlm.to_logits
    w64 = head.weight.detach().to(BF16).double().requires_grad_(True)    # the kernel's operand
    b64 = head.bias.detach().double().requires_grad_(True)
    ref = F.cross_entropy(F.linear(enc[sel].double(), w64, b64), labels[sel])
    ref.backward()
    assert abs(loss.item() - ref.item()) <= LOSS_GATE * abs(ref.item()) + 1e-6
    assert _rel(head.weight.grad, w64.grad) <= DW_GATE
    assert _rel(head.bias.grad, b64.grad) <= DB_GATE
    assert clip.text_transformer.token_emb.weight.grad.abs().sum() > 0
