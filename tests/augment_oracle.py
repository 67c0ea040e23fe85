"""The reference's SimCLR augmentation as torchvision builds it (x_clip/visual_ssl.py:24-45, :59-88): the
`nn.Sequential` that `aux.default_augmentation` returned before the CUDA kernels, a recorder of the
parameters it applies (each functional op it calls, with its arguments), and augment64, the fp64
restatement of one kernels.augment call from that wrapper's own arguments."""
import torch
import torch.nn.functional as F
from torch import nn
from torchvision import transforms as T
from torchvision.transforms import functional as TF

# max |kernel - fp64| over max(1, max |fp64|) of one call; about twice the largest error measured on an
# H100 (8.5e-6, 3 x 130 x 97 -> 224: the resample's fp32 weights, which ATen's fp32 path computes the
# same way).  Shared by test_gpu_augment.py and the per-call check of bench_call_oracle.py.
GATE = 2e-5
GRAY = (0.2989, 0.587, 0.114)           # torchvision's rgb_to_grayscale weights


def _gray(x):
    return (GRAY[0] * x[:, 0] + GRAY[1] * x[:, 1] + GRAY[2] * x[:, 2]).unsqueeze(1)


def _blend(x, other, f, om):
    """torchvision's _blend for float images: clamp(f x + (1 - f) other, 0, 1), (1 - f) as passed."""
    return (f * x + om * other).clamp(0.0, 1.0)


def augment64(x, *, ops=(), factor=(0.0,) * 4, one_minus=(0.0,) * 4, grayscale=False, flip=False,
              blur_kernel=None, normalize=None, crop, out_size):
    """kernels.augment(x, ...) in float64, from the wrapper's arguments: the jitter ops in order
    (brightness, contrast against each image's grey mean, saturation, torchvision's hue), grayscale,
    horizontal flip, the 3 x 3 blur_kernel (row-major) with reflect padding, the crop (top, left, height,
    width) resampled to out_size by torchvision's antialiased bilinear resize, then normalize."""
    x = x.double()
    C = x.shape[1]
    for op in ops:
        f, om = float(factor[op]), float(one_minus[op])
        if op == 0:
            x = _blend(x, torch.zeros_like(x), f, om)
        elif op == 1:
            x = _blend(x, _gray(x).mean(dim=(-3, -2, -1), keepdim=True), f, om)
        elif op == 2:
            x = _blend(x, _gray(x), f, om)
        else:
            x = TF.adjust_hue(x, f)
    if grayscale:
        x = _gray(x).expand(-1, C, -1, -1)
    if flip:
        x = x.flip(-1)
    if blur_kernel is not None:
        k = torch.tensor([float(w) for w in blur_kernel], dtype=torch.float64, device=x.device).view(1, 1, 3, 3)
        x = F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), k.expand(C, 1, 3, 3), groups=C)
    top, left, h, w = (int(v) for v in crop)
    x = TF.resized_crop(x, top, left, h, w, [int(v) for v in out_size], TF.InterpolationMode.BILINEAR,
                        antialias=True)
    if normalize is not None:
        mean = torch.tensor(normalize[0], dtype=torch.float64, device=x.device).view(1, -1, 1, 1)
        std = torch.tensor(normalize[1], dtype=torch.float64, device=x.device).view(1, -1, 1, 1)
        x = (x - mean) / std
    return x


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
