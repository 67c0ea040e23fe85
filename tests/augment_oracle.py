"""The reference's SimCLR augmentation as torchvision builds it (x_clip/visual_ssl.py:24-45, :59-88): the
`nn.Sequential` that `aux.default_augmentation` returned before the CUDA kernels, and a recorder of the
parameters it applies (each functional op it calls, with its arguments)."""
import torch
from torch import nn
from torchvision import transforms as T
from torchvision.transforms import functional as TF


class RandomApply(nn.Module):
    def __init__(self, fn, p):
        super().__init__()
        self.fn, self.p = fn, p

    def forward(self, x):
        return x if torch.rand(()) > self.p else self.fn(x)


def torchvision_augmentation(image_size: int, channels: int = 3) -> nn.Module:
    is_rgb = channels == 3
    is_gt1 = channels > 1
    return nn.Sequential(
        RandomApply(T.ColorJitter(0.8, 0.8, 0.8, 0.2), p=0.3) if is_rgb else nn.Identity(),
        T.RandomGrayscale(p=0.2) if is_rgb else nn.Identity(),
        T.RandomHorizontalFlip(),
        RandomApply(T.GaussianBlur((3, 3), (1.0, 2.0)), p=0.2) if is_gt1 else nn.Identity(),
        T.RandomResizedCrop((image_size, image_size)),
        T.Normalize(mean=torch.tensor([0.485, 0.456, 0.406]), std=torch.tensor([0.229, 0.224, 0.225]))
        if is_rgb else nn.Identity(),
    )


_JITTER = {"adjust_brightness": 0, "adjust_contrast": 1, "adjust_saturation": 2, "adjust_hue": 3}


def record(monkeypatch):
    """Wrap the functional ops the transforms call; -> the list the Sequential's calls append to:
    ("jitter", op id, factor), ("grayscale",), ("flip",), ("blur", sigma), ("crop", (i, j, h, w))."""
    calls = []

    def wrap(name, entry):
        real = getattr(TF, name)

        def fn(*args, **kw):
            calls.append(entry(args))
            return real(*args, **kw)
        monkeypatch.setattr(TF, name, fn)

    for name, op in _JITTER.items():
        wrap(name, lambda a, op=op: ("jitter", op, a[1]))
    wrap("rgb_to_grayscale", lambda a: ("grayscale",))
    wrap("hflip", lambda a: ("flip",))
    wrap("gaussian_blur", lambda a: ("blur", a[2][0]))
    wrap("resized_crop", lambda a: ("crop", tuple(a[1:5])))
    return calls


def expected_calls(params):
    """The calls the Sequential makes for SimCLRAugmentation params."""
    out = [("jitter", op, params.factors[op]) for op in params.order]
    if params.grayscale:
        out.append(("grayscale",))
    if params.flip:
        out.append(("flip",))
    if params.sigma is not None:
        out.append(("blur", params.sigma))
    out.append(("crop", params.crop))
    return out
