"""Float64 CPU restatement of LPIPS (lpips v0.1, net='vgg', lpips=True, spatial=False), the yardstick of aphantasia_b200.lpips.

    x <- 2x - 1 (normalize=True);  x <- (x - shift) / scale
    torchvision vgg16().features[0:30], taps after indices 3, 8, 15, 22, 29 (relu1_2 ... relu5_3)
    n = f / (sqrt(sum_c f^2) + 1e-10);  value = sum_taps mean_{h,w} sum_c lin[c] (n0 - n1)^2          -> [N,1,1,1]

The norm is written as sqrt(sum of squares), as lpips writes it, so its autograd gradient at an all-zero pixel is NaN, and the
ReLU backward (a select) removes it exactly as it does upstream.
"""
import torch

SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
TAPS = (3, 8, 15, 22, 29)


class _RoundBF16(torch.autograd.Function):
    """Rounds to bf16 in the forward and the gradient to bf16 in the backward (float64 in between)."""
    @staticmethod
    def forward(ctx, x):
        return x.to(torch.bfloat16).double()

    @staticmethod
    def backward(ctx, g):
        return g.to(torch.bfloat16).double()


def vgg_features(vgg_sd, bf16=False):
    """torchvision's vgg16(weights=None).features[0:30] in float64 with the conv weights of `vgg_sd` (features.{i}.*). The
    global RNG (torchvision initialises before the load) is restored. bf16=True: the weights of every conv but the first are
    rounded to bf16, as the CUDA path packs them."""
    import torchvision
    with torch.random.fork_rng(devices=[]):
        feats = torchvision.models.vgg16(weights=None).features[:30].double().eval()
    sd = {k[len('features.'):]: v.double() for k, v in vgg_sd.items() if k.startswith('features.')}
    if bf16:
        sd = {k: (v.to(torch.bfloat16).double() if k.endswith('weight') and not k.startswith('0.') else v) for k, v in sd.items()}
    feats.load_state_dict(sd)
    for p in feats.parameters():
        p.requires_grad_(False)
    return feats


def taps(feats, x, bf16=False):
    """bf16=True: every ReLU output is rounded to bf16, and its gradient too (where the CUDA path stores them)."""
    out = []
    for i, layer in enumerate(feats):
        x = layer(x)
        if bf16 and isinstance(layer, torch.nn.ReLU):
            x = _RoundBF16.apply(x)
        if i in TAPS:
            out.append(x)
    return out


def lpips(in0, in1, vgg_sd, lin_sd, normalize=True, feats=None, bf16=False):
    """float64 [N,1,1,1] on in0's device (the GPU tests run it there in float64); differentiable in in0.
    bf16=True is the rounding model of the CUDA path: bf16 weights (conv1_1 excepted), bf16 activations and activation
    gradients, everything else float64. It moves the max-pool argmaxes and ReLU masks where the CUDA path moves them."""
    feats = (feats if feats is not None else vgg_features(vgg_sd, bf16)).to(in0.device)
    shift = torch.tensor(SHIFT, dtype=torch.float64, device=in0.device).view(1, 3, 1, 1)
    scale = torch.tensor(SCALE, dtype=torch.float64, device=in0.device).view(1, 3, 1, 1)

    def prep(x):
        x = x.double()
        if normalize:
            x = 2 * x - 1
        return (x - shift) / scale

    f0s, f1s = taps(feats, prep(in0), bf16), taps(feats, prep(in1), bf16)
    val = 0
    for t, (f0, f1) in enumerate(zip(f0s, f1s)):
        n0 = f0 / (torch.sqrt(torch.sum(f0 ** 2, dim=1, keepdim=True)) + 1e-10)
        n1 = f1 / (torch.sqrt(torch.sum(f1 ** 2, dim=1, keepdim=True)) + 1e-10)
        w = lin_sd['lin%d.model.1.weight' % t].double().to(in0.device)
        d = torch.nn.functional.conv2d((n0 - n1) ** 2, w)
        val = val + d.mean(dim=[2, 3], keepdim=True)
    return val
