"""ViT-B/16, -B/32, -L/16 and -L/32 on CPU: torchvision parity (state_dict keys, order and shapes, parameter counts,
image_size, unsupported builder arguments, initialisation, eval logits, and vit_b_32's train-mode logits, every
parameter gradient and the input gradient against float64), the encoder-block and self-attention composites against
torchvision's ``EncoderBlock`` and ``nn.MultiheadAttention``, the attention predicate and the new kernels' ptxas
figures."""
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F
import torchvision
from torchvision.models.vision_transformer import EncoderBlock as TvEncoderBlock

from distributeddeeplearning_b200 import _ext, models, ops
from distributeddeeplearning_b200.models.vit import EncoderBlock
from distributeddeeplearning_b200.ops import native

NAMES = ["vit_b_16", "vit_b_32", "vit_l_16", "vit_l_32"]
PARAMS = dict(zip(NAMES, [86_567_656, 88_224_232, 304_326_632, 306_535_400]))


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_order_shapes_and_parameter_counts_match_torchvision(name):
    m = models.get_model(name)
    tv = getattr(torchvision.models, name)()
    assert list(m.state_dict()) == list(tv.state_dict())
    assert [tuple(v.shape) for v in m.state_dict().values()] == [tuple(v.shape) for v in tv.state_dict().values()]
    assert [k for k, _ in m.named_parameters()] == [k for k, _ in tv.named_parameters()]
    assert sum(p.numel() for p in m.parameters()) == sum(p.numel() for p in tv.parameters()) == PARAMS[name]
    assert models.input_size(m) == models.input_size(name) == 224
    lns = [mod for mod in m.modules() if isinstance(mod, models.layers.LayerNorm)]
    assert len(lns) == 2 * len(m.encoder.layers) + 1 and all(ln.eps == 1e-6 for ln in lns)
    blk = m.encoder.layers[0]
    c = m.hidden_dim
    assert native.supports_attention(m.seq_length, blk.num_heads, c // blk.num_heads)
    assert native.supports_layer_norm(c)


def test_image_size_and_unsupported_builder_arguments():
    m, tv = models.get_model("vit_b_16", image_size=384), torchvision.models.vit_b_16(image_size=384)
    assert m.seq_length == 577 and m.input_size == models.input_size(m) == 384
    assert m.encoder.pos_embedding.shape == tv.encoder.pos_embedding.shape == (1, 577, 768)
    m = models.get_model("vit_b_32", image_size=384, num_classes=10)
    assert m.seq_length == 145 and m.heads.head.out_features == 10
    assert sum(p.numel() for p in models.get_model("vit_b_32", image_size=384).parameters()) == 88_297_192
    for kw in (dict(dropout=0.1), dict(attention_dropout=0.1), dict(representation_size=768),
               dict(conv_stem_configs=[]), dict(image_size=200), dict(pretrained=True)):
        with pytest.raises(ValueError):
            models.get_model("vit_b_32", **kw)


def test_initialisation_follows_torchvision():
    torch.manual_seed(0)
    m, tv = models.get_model("vit_b_16"), torchvision.models.vit_b_16()
    for k, p in m.state_dict().items():
        q = tv.state_dict()[k]
        if k in ("class_token", "conv_proj.bias", "heads.head.weight", "heads.head.bias") or \
                k.endswith("in_proj_bias") or k.endswith("out_proj.bias"):
            assert torch.equal(p, torch.zeros_like(p)) and torch.equal(q, torch.zeros_like(q)), k
        elif re.search(r"ln(_\d)?\.weight$", k):
            assert torch.equal(p, torch.ones_like(p)), k
        elif re.search(r"ln(_\d)?\.bias$", k):
            assert torch.equal(p, torch.zeros_like(p)), k
        else:                                # random: same spread (and range) as torchvision's draw, within sampling noise
            tol = 0.02 + 4 / p.numel() ** 0.5
            assert abs(float(p.std()) / float(q.std()) - 1) < tol, k
            assert abs(float(p.mean())) < tol * float(q.std()), k
            if p.numel() > 100_000:
                assert abs(float(p.abs().max()) / float(q.abs().max()) - 1) < 0.25, k
    assert m.conv_proj.weight.is_contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("name", NAMES)
def test_eval_equals_torchvision(name):
    torch.manual_seed(0)
    size = 64 if name.endswith("32") else 32
    m = models.get_model(name, num_classes=10, image_size=size)
    tv = getattr(torchvision.models, name)(num_classes=10, image_size=size)
    with torch.no_grad():
        for p in tv.parameters():
            p.add_(torch.randn_like(p) * 0.02)       # perturbed LayerNorm affines and biases, a non-zero head
    m.load_state_dict(tv.state_dict())
    m.eval(), tv.eval()
    x = torch.randn(2, 3, size, size)
    with torch.no_grad():
        out, ref = m(x), tv(x)
    assert torch.allclose(out, ref, atol=1e-4, rtol=1e-4), float((out - ref).abs().max())


def test_b32_train_forward_backward_equals_float64_torchvision():
    torch.manual_seed(3)
    m, tv = models.get_model("vit_b_32"), torchvision.models.vit_b_32()
    with torch.no_grad():
        for name, p in tv.named_parameters():
            if p.dim() == 1 or name.startswith("heads") or name == "class_token":
                p.add_(torch.randn_like(p) * 0.1)
    m.load_state_dict(tv.state_dict())
    tv = tv.double()
    m.train(), tv.train()
    x = torch.randn(2, 3, 224, 224)
    xs, xd = x.clone().requires_grad_(True), x.double().requires_grad_(True)
    y = torch.tensor([1, 7])
    o1, o2 = m(xs), tv(xd)
    assert torch.allclose(o1.double(), o2, atol=1e-3, rtol=1e-3), float((o1.double() - o2).abs().max())
    ops.softmax_cross_entropy(o1, y).backward()
    F.cross_entropy(o2, y).backward()
    g1 = dict(m.named_parameters())
    for k, p in tv.named_parameters():
        err = float((g1[k].grad.double() - p.grad).norm() / max(float(p.grad.norm()), 1e-6))
        assert err < 1e-3, (k, err)
    err = float((xs.grad.double() - xd.grad).norm() / xd.grad.norm())
    assert err < 1e-3, err


@pytest.mark.parametrize("L", [5, 70])
def test_block_and_attention_composites_equal_torchvision_in_float64(L):
    torch.manual_seed(L)
    C, heads = 48, 4
    ref = TvEncoderBlock(heads, C, 96, 0.0, 0.0).double()
    with torch.no_grad():
        for p in ref.parameters():
            p.add_(torch.randn_like(p) * 0.2)
    blk = EncoderBlock(heads, C, 96).double()
    blk.load_state_dict(ref.state_dict())
    assert list(blk.state_dict()) == list(ref.state_dict())
    x = torch.randn(3, L, C, dtype=torch.float64, requires_grad=True)
    xr = x.detach().clone().requires_grad_(True)
    z, zr = blk(x), ref(xr)
    assert torch.allclose(z, zr, atol=1e-10, rtol=1e-10)
    g = torch.randn_like(z)
    z.backward(g)
    zr.backward(g)
    assert torch.allclose(x.grad, xr.grad, atol=1e-10, rtol=1e-10)
    for (k, p), (_, q) in zip(blk.named_parameters(), ref.named_parameters()):
        assert torch.allclose(p.grad, q.grad, atol=1e-10, rtol=1e-10), k
    # self_attention on the packed qkv against nn.MultiheadAttention with an identity in-projection
    mha = torch.nn.MultiheadAttention(C, heads, batch_first=True).double()
    with torch.no_grad():
        mha.in_proj_weight.copy_(torch.eye(C, dtype=torch.float64).repeat(3, 1))
        mha.in_proj_bias.zero_()
        mha.out_proj.weight.copy_(torch.eye(C, dtype=torch.float64))
        mha.out_proj.bias.zero_()
    q, k, v = (torch.randn(2, L, C, dtype=torch.float64) for _ in range(3))
    ref_o, _ = mha(q, k, v, need_weights=False)
    assert torch.allclose(ops.self_attention(torch.cat([q, k, v], dim=2), heads), ref_o, atol=1e-10, rtol=1e-10)


def test_supports_attention():
    assert native.supports_attention(197, 12, 64) and native.supports_attention(1, 16, 64)
    assert native.supports_attention(577, 12, 64) and native.supports_attention(50, 16, 64)
    assert not native.supports_attention(257, 16, 80)          # vit_h_14
    assert not native.supports_attention(0, 12, 64) and not native.supports_attention(197, 0, 64)


def _ptxas(src):
    """{demangled kernel name: (registers, spill store bytes, spill load bytes, stack bytes)} of one .cu file built for
    sm_90a."""
    nvcc = os.path.join(_ext.CUDA_HOME, "bin", "nvcc")
    csrc = os.path.join(os.path.dirname(_ext.__file__), "csrc")
    r = subprocess.run([nvcc, "-c", os.path.join(csrc, "ops", src), "-o", os.devnull, "-O3", "-std=c++17", *_ext.NVCC_ARCH,
                        "--expt-relaxed-constexpr", "-I", csrc, "-Xptxas", "-v"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    out, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            cur = re.sub(r"^(void )?ddl::|\(.*\)$", "", cur.replace("(anonymous namespace)::", ""))
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = [0, int(m.group(2)), int(m.group(3)), int(m.group(1))]
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            out[cur][0] = int(m.group(1))
    return out


_NVCC = shutil.which("c++filt") and os.path.isfile(os.path.join(_ext.CUDA_HOME, "bin", "nvcc"))


@pytest.mark.skipif(not _NVCC, reason="needs nvcc and c++filt")
def test_new_kernels_compile_without_spills_and_fit_their_launch_bounds():
    at = _ptxas("attention.cu")
    assert sorted(at) == ["attn_bwd_dkv_kernel", "attn_bwd_dq_kernel", "attn_fwd_kernel"], sorted(at)
    for n, (regs, st, ld, stack) in at.items():
        assert st == 0 and ld == 0 and stack == 0 and regs <= 255, (n, regs, st, ld, stack)   # 128 threads
    vt = _ptxas("vit.cu")
    assert len(vt) == 16, sorted(vt)   # add+LN fwd / LN bwd with addend for V = 1..6, patchify, tokens fwd / bwd / reduce
    for n, (regs, st, ld, stack) in vt.items():
        v = re.search(r"<(\d+)>", n)
        bound = 255
        if v and "fwd" in n and int(v.group(1)) <= 5 or v and "bwd" in n and int(v.group(1)) <= 3:
            bound = 128                         # two blocks of 256 threads per SM
        assert st == 0 and ld == 0 and regs <= bound, (n, regs, st, ld)
