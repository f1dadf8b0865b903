"""One forward for several ViT layers (dvt_vit_forward_layers) against one dvt_vit_forward per layer: `torch.equal` for
every backbone family (DINOv2-S reg4, the pre-norm CLIP tower, ViT-H/14 at head_dim 80, DINOv3-S with RoPE, the SwiGLU
ViT-g, each at reduced depth), with and without the final norm and the prefix tokens, NCHW and NLC, `n` as an int and as
unsorted, repeated and negative indices, batch 1 and 3, non-square inputs, a stride below the patch size, on the
tensor-core and the SIMT path.  Also the channel-concatenated buffer of the probes against torch.cat of the per-layer maps,
its cls rows against prefix token 0 of each layer, and the refusals that need a handle."""
import contextlib
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

DEPTH = 4
# (identifier, arch table, patch, the two input cases: (B, H, W, stride))
BACKBONES = {
    "dinov2-s-reg4": ("vit_small_patch14_reg4_dinov2.lvd142m", "ARCHS", 14, [(1, 56, 56, 14), (3, 70, 98, 7)]),
    "clip-b16": ("vit_base_patch16_clip_224.openai", "ARCHS", 16, [(1, 64, 64, 16), (3, 64, 96, 8)]),
    "vith14-hd80": ("vit_huge_patch14_224.mae", "ARCHS", 14, [(1, 56, 56, 14), (3, 56, 84, 10)]),
    "dinov3-s-rope": ("vit_small_patch16_dinov3.lvd1689m", "DINOV3_ARCHS", 16, [(1, 64, 64, 16), (3, 64, 96, 12)]),
    "vitg14-swiglu": ("vit_giant_patch14_dinov2.lvd142m", "ARCHS", 14, [(1, 56, 56, 14), (3, 42, 70, 7)]),
}
# the forms of `n` of get_intermediate_layers, at depth 4
N_FORMS = {"int": 3, "unsorted": [3, 0, 2], "repeated": [1, 3, 1], "negative": [-1, 0, -3], "last": [3]}


@contextlib.contextmanager
def _impl(impl):
    from dvt import _lib
    _lib.check(_lib.lib().dvt_set_debug_impl(impl), "dvt_set_debug_impl")
    try:
        yield
    finally:
        _lib.lib().dvt_set_debug_impl(-1)


def _dev_ok():
    from dvt import _lib
    torch.cuda.synchronize()
    assert _lib.device_error() == 0


_MODELS = {}


def _model(name):
    """B200VisionTransformer of `name` at depth 4 with every parameter randomised (LayerNorms and LayerScales included, so
    that the layers differ), on cuda."""
    if name not in _MODELS:
        from dvt.models import vit_wrapper as VW
        ident, table, patch, _ = BACKBONES[name]
        a = dict(getattr(VW, table)[ident], depth=DEPTH)
        torch.manual_seed(0)
        m = VW.B200VisionTransformer(ident, patch, a)
        with torch.no_grad():
            for p in m.parameters():
                p.add_(torch.randn_like(p) * 0.05)
        _MODELS[name] = m.cuda().eval()
    return _MODELS[name]


def _input(B, H, W, seed=1):
    return torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(seed + B + H + W)).cuda()


def _take(n):
    return list(range(DEPTH - n, DEPTH)) if isinstance(n, int) else [i % DEPTH for i in n]


@pytest.mark.parametrize("impl", [0, 1], ids=["tc", "simt"])
@pytest.mark.parametrize("name", list(BACKBONES))
def test_one_pass_equals_one_forward_per_layer(name, impl):
    m = _model(name)
    npre = m.num_prefix_tokens
    with _impl(impl):
        for case in BACKBONES[name][3]:
            B, H, W, stride = case
            m.patch_embed.proj.stride = [stride, stride]
            x = _input(B, H, W)
            h, w = (H - m.patch_embed.patch_size[0]) // stride + 1, (W - m.patch_embed.patch_size[0]) // stride + 1
            for norm in (False, True):
                ref = {i: m._run(x, i, norm, all_tokens=True) for i in range(DEPTH)}   # dvt_vit_forward per layer
                assert not torch.equal(ref[0], ref[DEPTH - 1])
                for prefix in (False, True):
                    for fmt in ("NCHW", "NLC"):
                        for form, n in N_FORMS.items():
                            what = (case, norm, prefix, fmt, form)
                            outs = m.forward_intermediates(x, n, return_prefix_tokens=prefix, norm=norm, output_fmt=fmt,
                                                           intermediates_only=True)
                            take = _take(n)
                            assert len(outs) == len(take), what
                            storages = set()
                            for idx, o in zip(take, outs):
                                feat, pre = o if prefix else (o, None)
                                want = ref[idx][:, npre:]
                                if fmt == "NCHW":
                                    assert feat.shape == (B, m.embed_dim, h, w), what
                                    feat = feat.permute(0, 2, 3, 1).reshape(B, h * w, -1)
                                else:
                                    assert feat.shape == (B, h * w, m.embed_dim), what
                                assert torch.equal(feat, want), what
                                if prefix:
                                    assert torch.equal(pre, ref[idx][:, :npre]), what
                                else:   # NCHW: a view of the layer's own contiguous NHWC tensor
                                    assert fmt == "NLC" or o.permute(0, 2, 3, 1).is_contiguous(), what
                                storages.add(feat.untyped_storage().data_ptr())
                            assert len(storages) == len(take), what   # repeated layers do not share a tensor
    m.patch_embed.proj.stride = [m.patch_embed.patch_size[0]] * 2
    _dev_ok()


@pytest.mark.parametrize("impl", [0, 1], ids=["tc", "simt"])
@pytest.mark.parametrize("name", ["dinov2-s-reg4", "dinov3-s-rope", "clip-b16"])
def test_concatenated_maps_and_cls_rows(name, impl):
    m = _model(name)
    npre = m.num_prefix_tokens
    with _impl(impl):
        for B, H, W, stride in BACKBONES[name][3]:
            m.patch_embed.proj.stride = [stride, stride]
            x = _input(B, H, W, seed=5)
            for norm in (False, True):
                maps = {i: m._run(x, i, norm, all_tokens=False) for i in range(DEPTH)}
                tokens = {i: m._run(x, i, norm, all_tokens=True) for i in range(DEPTH)}
                for layers in ([0, 1, 2, 3], [1, 3], [3], [3, 0, 2], [2, 2, -1]):
                    ls = [i % DEPTH for i in layers]
                    cat, cls = m.forward_layers_concat(x, layers, norm=norm, return_cls=True)
                    assert cat.is_contiguous() and cat.shape[-1] == len(ls) * m.embed_dim
                    assert torch.equal(cat, torch.cat([maps[i] for i in ls], -1)), (layers, norm)
                    assert torch.equal(cls, torch.cat([tokens[i][:, 0] for i in ls], -1)), (layers, norm)
                    assert torch.equal(m.forward_layers_concat(x, layers, norm=norm), cat)
            # every prefix row of a tap, registers included, against the all-tokens forward
            for norm in (False, True):
                _, pre = m._run_layers(x, [1, 3], norm, concat=True, prefix=True)
                for l, i in enumerate([1, 3]):
                    assert torch.equal(pre[l], m._run(x, i, norm, all_tokens=True)[:, :npre])
    m.patch_embed.proj.stride = [m.patch_embed.patch_size[0]] * 2
    _dev_ok()


def test_refusals_that_need_the_handle():
    from dvt import _lib
    m = _model("dinov2-s-reg4")
    x = _input(1, 56, 56)
    x, stride, h, w, pos_patch, prefix_rows, rope = m._prep(x)
    C = m.embed_dim
    out = torch.empty(1, h, w, 2 * C, device="cuda")

    def call(layers, ldo):
        n = len(layers)
        ptrs = (ctypes.c_void_p * n)(*[out.data_ptr() + 4 * C * l for l in range(n)])
        return _lib.lib().dvt_vit_forward_layers(m._handle, _lib.ptr(x), _lib.DT_F32, 1, 56, 56, stride, _lib.ptr(pos_patch),
                                                 _lib.ptr(prefix_rows), None, n, (ctypes.c_int * n)(*layers), 0, ptrs, ldo,
                                                 0, None, _lib.cur_stream())

    assert call([1, DEPTH], 2 * C) == 1 and f"layer_indices[1]={DEPTH} out of range [0, {DEPTH})" in \
        _lib.lib().dvt_last_error().decode()
    assert call([1, 2], C - 4) == 1 and f"ldo={C - 4} must be >= C={C}" in _lib.lib().dvt_last_error().decode()
    assert call([1, 2], 2 * C) == 0
    _dev_ok()
    assert torch.equal(out[..., C:], m._run(x, 2, False, all_tokens=False))
