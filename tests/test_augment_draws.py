"""SimCLRAugmentation.draw against the torchvision Sequential it replaces (CPU): the same draws from the
CPU generator, in the same order, and no parameters or buffers in the model's state."""
import pytest
import torch

import augment_oracle as AO
from x_clip_b200.aux import SimCLRAugmentation

SHAPES = [(2, 16, 16), (1, 33, 65), (3, 7, 40), (2, 64, 31), (5, 2, 2)]


@pytest.mark.parametrize("channels", [1, 3, 4])
def test_draw_matches_the_sequential(monkeypatch, channels):
    """Over 300 seeds and 5 shapes: the CPU generator's state after `draw` equals the one the Sequential
    leaves after augmenting a CPU tensor of that shape, and `draw` returns what the Sequential applied."""
    calls = AO.record(monkeypatch)
    seen = set()
    for seed in range(300):
        b, h, w = SHAPES[seed % len(SHAPES)]
        size = max(h, w)
        seq = AO.torchvision_augmentation(size, channels)
        aug = SimCLRAugmentation(size, channels)
        x = torch.rand(b, channels, h, w)
        torch.manual_seed(seed)
        calls.clear()
        seq(x)
        state = torch.get_rng_state()
        torch.manual_seed(seed)
        p = aug.draw(x.shape)
        assert torch.equal(torch.get_rng_state(), state), (seed, channels)
        assert calls == AO.expected_calls(p), (seed, channels, calls, p)
        seen.add((bool(p.order), p.grayscale, p.flip, p.sigma is not None))
    # every branch was taken both ways
    for k in range(4):
        vals = {s[k] for s in seen}
        if channels != 3 and k < 2:
            assert vals == {False}
        elif channels == 1 and k == 3:
            assert vals == {False}
        else:
            assert vals == {False, True}, (k, channels)


@pytest.mark.parametrize("ssl_type", ["simsiam", "simclr"])
def test_state_dict_keys_unchanged(ssl_type):
    """The augmentation registers nothing: the keys equal those of the model with the torchvision
    Sequential in its place."""
    import x_clip_b200
    kw = dict(dim_text=256, dim_image=256, dim_latent=256, num_text_tokens=128, text_enc_depth=1,
              text_seq_len=16, text_heads=4, visual_enc_depth=1, visual_heads=4, visual_image_size=64,
              visual_patch_size=16, use_visual_ssl=True, visual_ssl_type=ssl_type)
    clip = x_clip_b200.CLIP(**kw)
    ssl = clip.visual_ssl
    assert isinstance(ssl.augment1, SimCLRAugmentation) and ssl.augment2 is ssl.augment1
    assert not list(ssl.augment1.parameters()) and not list(ssl.augment1.buffers())
    keys = list(clip.state_dict().keys())
    ssl.augment1 = ssl.augment2 = AO.torchvision_augmentation(64, 3)
    assert keys == list(clip.state_dict().keys())


def test_user_augmentations_are_kept():
    from x_clip_b200.aux import SimCLR, SimSiam
    net = torch.nn.Linear(4, 4)
    f1, f2 = torch.nn.Identity(), torch.nn.Identity()
    for cls in (SimSiam, SimCLR):
        m = cls(net, 64, rep_dim=4, augment_fn=f1, augment_fn2=f2)
        assert m.augment1 is f1 and m.augment2 is f2


def test_cpu_input_takes_torchvision():
    """A CPU input (and any input that requires grad) takes the functional ops with the drawn
    parameters: the Sequential's result from the same seed."""
    seq, aug = AO.torchvision_augmentation(24, 3), SimCLRAugmentation(24, 3)
    x = torch.rand(2, 3, 24, 24)
    for seed in range(20):
        torch.manual_seed(seed)
        ref = seq(x)
        torch.manual_seed(seed)
        assert torch.equal(aug(x), ref), seed
