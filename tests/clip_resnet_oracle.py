"""Float64 restatement of CLIP's ModifiedResNet image tower in eval mode, from an OpenAI-layout state dict (keys without the
"visual." prefix): F.conv2d, F.batch_norm on the running statistics (eps 1e-5), F.avg_pool2d and F.multi_head_attention_forward.
Its gradient is taken by autograd. Written from the architecture; it shares no code with the CUDA tower.

`selects` replaces every ReLU by a given select: a list of boolean NCHW tensors in the order the CUDA tower saves its ReLU outputs
(the stem's three, then each block's conv1, conv2 and output), each True where that ReLU output is > 0. With the CUDA forward's
own selects the tower is linear in its input up to the attention pool, so its backward differs from the CUDA one by rounding
only, not by the ReLUs that bf16 activations flip. `pool_input` (the CUDA tower's last block output, NCHW) replaces the values the
attention pool reads while its gradient still flows into this restatement's own trunk: the attention pool's softmax is not linear,
and its gradient then sees the CUDA forward's inputs rather than float64 ones. `dtype` runs the same ops in another precision
(profiles: eager fp16)."""
import torch
import torch.nn.functional as F


class _Relu:
    def __init__(self, selects):
        self.selects, self.i = selects, 0

    def __call__(self, x):
        if self.selects is None:
            return F.relu(x)
        m = self.selects[self.i]
        self.i += 1
        assert m.shape == x.shape, (self.i - 1, tuple(m.shape), tuple(x.shape))
        return torch.where(m, x, torch.zeros_like(x))


def _bn(x, sd, p):
    dt = x.dtype
    return F.batch_norm(x, sd[p + '.running_mean'].to(dt), sd[p + '.running_var'].to(dt), sd[p + '.weight'].to(dt),
                        sd[p + '.bias'].to(dt), training=False, eps=1e-5)


def _conv(x, sd, k, stride=1, pad=0):
    return F.conv2d(x, sd[k].to(x.dtype), stride=stride, padding=pad)


def _bottleneck(x, sd, p, stride, relu):
    out = relu(_bn(_conv(x, sd, p + 'conv1.weight'), sd, p + 'bn1'))
    out = relu(_bn(_conv(out, sd, p + 'conv2.weight', pad=1), sd, p + 'bn2'))
    if stride > 1:
        out = F.avg_pool2d(out, stride)
    out = _bn(_conv(out, sd, p + 'conv3.weight'), sd, p + 'bn3')
    idt = x
    if p + 'downsample.0.weight' in sd:
        idt = F.avg_pool2d(x, stride) if stride > 1 else x
        idt = _bn(_conv(idt, sd, p + 'downsample.0.weight'), sd, p + 'downsample.1')
    return relu(out + idt)


def forward(sd, x, selects=None, dtype=torch.float64, pool_input=None):
    """x [S,3,side,side] -> embeddings [S, out_dim], in `dtype`."""
    relu = _Relu(selects)
    x = x.to(dtype)
    x = relu(_bn(_conv(x, sd, 'conv1.weight', stride=2, pad=1), sd, 'bn1'))
    x = relu(_bn(_conv(x, sd, 'conv2.weight', pad=1), sd, 'bn2'))
    x = relu(_bn(_conv(x, sd, 'conv3.weight', pad=1), sd, 'bn3'))
    x = F.avg_pool2d(x, 2)
    for i in range(1, 5):
        n = len({k.split('.')[1] for k in sd if k.startswith('layer%d.' % i)})
        for j in range(n):
            x = _bottleneck(x, sd, 'layer%d.%d.' % (i, j), 2 if (i > 1 and j == 0) else 1, relu)
    if pool_input is not None:
        x = x + (pool_input.to(dtype) - x).detach()
    S, Cc, H, W = x.shape
    t = x.reshape(S, Cc, H * W).permute(2, 0, 1)                       # (HW, S, C)
    t = torch.cat([t.mean(dim=0, keepdim=True), t], dim=0)
    t = t + sd['attnpool.positional_embedding'].to(dtype)[:, None, :]
    a = 'attnpool.'
    d = lambda k: sd[a + k].to(dtype)
    out, _ = F.multi_head_attention_forward(
        query=t[:1], key=t, value=t, embed_dim_to_check=Cc, num_heads=Cc // 64,
        q_proj_weight=d('q_proj.weight'), k_proj_weight=d('k_proj.weight'), v_proj_weight=d('v_proj.weight'), in_proj_weight=None,
        in_proj_bias=torch.cat([d('q_proj.bias'), d('k_proj.bias'), d('v_proj.bias')]), bias_k=None, bias_v=None,
        add_zero_attn=False, dropout_p=0., out_proj_weight=d('c_proj.weight'), out_proj_bias=d('c_proj.bias'),
        use_separate_proj_weight=True, training=False, need_weights=False)
    assert selects is None or relu.i == len(selects)
    return out.squeeze(0)


def forward_backward(sd, x, g, selects=None, pool_input=None):
    """(embeddings, d <embeddings, g> / d x) in float64."""
    xi = x.double().clone().requires_grad_(True)
    e = forward(sd, xi, selects, pool_input=pool_input)
    (gx,) = torch.autograd.grad(e, xi, g.double())
    return e.detach(), gx
