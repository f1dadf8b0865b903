"""Stage-2 `Denoiser` forward on the GPU (SURVEY 8(f-4), inference): against the CPU oracle on feature-map input, with
a resampled position embedding, with two blocks, and end to end behind the frozen ViT.  Tolerance: cosine >= 0.999 per
patch (bf16 tensor-core GEMMs / attention against the fp32 oracle)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _min_cos(a, b):
    return F.cosine_similarity(a.float().flatten(0, -2), b.float().flatten(0, -2), dim=-1).min().item()


@pytest.mark.parametrize("nb,hw_in", [(1, (5, 6)), (2, (5, 6)), (1, (7, 9))], ids=["one-block", "two-blocks", "resampled-pe"])
def test_denoiser_forward_matches_oracle(nb, hw_in):
    import dvt.models as DVT
    from dvt import _lib
    from oracle import denoiser as OD
    C, hw = 128, (5, 6)
    sd = OD.random_state_dict(C, hw, nb, seed=nb)
    m = DVT.Denoiser(hw[0], hw[1], C, vit=None, enable_pe=True, num_blocks=nb)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    x = torch.randn(3, hw_in[0], hw_in[1], C, generator=torch.Generator().manual_seed(2))
    ref = OD.forward(sd, x, hw, nb)
    with torch.no_grad():
        got = m(x.cuda())
        d = m(x.cuda(), return_dict=True, return_channel_first=True)
    torch.cuda.synchronize()
    assert _lib.device_error() == 0
    assert got.shape == ref.shape and _min_cos(got.cpu(), ref) > 0.999
    assert (got.cpu() - ref).abs().max().item() < 0.08 * ref.abs().max().item()
    assert d["denoised_feats"].shape == (3, C, hw_in[0], hw_in[1]) and d["class_tokens"] is None
    assert torch.equal(d["original_feats"].cpu(), x)
    with pytest.raises(_lib.DvtError):
        m(x)                                     # CPU tensor: no fallback


def test_denoiser_behind_the_frozen_vit():
    import dvt.models as DVT
    from oracle import denoiser as OD
    from oracle import vit as OV
    ident = "vit_small_patch14_dinov2.lvd142m"
    torch.manual_seed(0)
    vit = DVT.PretrainedViTWrapper(ident, stride=14, allow_random_init=True)
    with torch.no_grad():
        for b in vit.model.blocks:
            b.ls1.gamma.uniform_(0.5, 1.5)
            b.ls2.gamma.uniform_(0.5, 1.5)
    C, hw = vit.n_output_dims, (5, 6)
    sd = OD.random_state_dict(C, hw, 1, seed=9)
    m = DVT.Denoiser(hw[0], hw[1], C, vit=vit, enable_pe=True)
    m.load_state_dict({**sd, **{"vit." + k: v for k, v in vit.state_dict().items()}}, strict=True)
    assert not any(p.requires_grad for p in m.vit.parameters())
    m = m.cuda().eval()
    x = torch.randn(2, 3, 70, 84, generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        got, cls = m(x.cuda(), return_class_token=True)
    cfg = OV.CONFIGS[ident]
    vsd = {k: v.detach().float().cpu() for k, v in vit.model.state_dict().items()}
    feats, prefix = OV.forward_intermediates(vsd, cfg, x, [cfg.depth - 1], stride=14, return_prefix_tokens=True)[0]
    ref = OD.forward(sd, feats.permute(0, 2, 3, 1), hw)
    assert got.shape == (2, 5, 6, C) and cls.shape == (2, C)
    assert _min_cos(got.cpu(), ref) > 0.999
    assert _min_cos(cls.cpu()[:, None], prefix[:, :1]) > 0.999


def test_long_sequence_attention():
    """N = 25 321 tokens (ViT at stride 4 on a 490 x 854 frame, make_video_demo.py:21-22,120): 198 key tiles per query tile
    through the flash-attention kernel against torch SDPA in fp32 on the same GPU."""
    from dvt import _lib, ops
    B, N, heads = 1, 25321, 2
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = (torch.randn(B, N, 3 * heads * 64, device="cuda", generator=g) * 1.5).bfloat16()
    out = ops.attention(qkv, heads)
    q, k, v = qkv.float().reshape(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4).unbind(0)
    ref = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, N, heads * 64)
    torch.cuda.synchronize()
    assert _lib.device_error() == 0
    assert (out.float() - ref).abs().max().item() < 3e-2
    assert _min_cos(out, ref) > 0.9995


def test_denoised_backbone_at_stride4_with_center_padding():
    """What SURVEY.md row f-4 is for: a video-sized frame (480 x 850) centre-padded to patch multiples (490 x 854), the
    frozen ViT at stride 4 -> 120 x 211 = 25 320 patch tokens, the learnable 37 x 37 position embedding resampled to that
    grid, one denoiser block over the 25 320-token sequence.  Checker: the oracle (ViT + Denoiser restatement) evaluated in
    fp32 on the same GPU (its explicit attention matrix needs ~30 GB: fine on a H100, not on a CPU box)."""
    import dvt.models as DVT
    from dvt import _lib
    from oracle import denoiser as OD
    from oracle import vit as OV
    ident = "vit_small_patch14_dinov2.lvd142m"
    cfg = OV.CONFIGS[ident]
    vsd = OV.random_state_dict(cfg, seed=5)
    vit = DVT.PretrainedViTWrapper(ident, stride=4, allow_random_init=True)
    vit.model.load_state_dict(vsd)
    C, hw = vit.n_output_dims, (37, 37)
    sd = OD.random_state_dict(C, hw, 1, seed=6)
    m = DVT.Denoiser(hw[0], hw[1], C, vit=vit, enable_pe=True)
    m.load_state_dict({**sd, **{"vit." + k: v for k, v in vit.state_dict().items()}}, strict=True)
    m = m.cuda().eval()
    frame = torch.randn(1, 3, 480, 850, generator=torch.Generator().manual_seed(7))
    x = DVT.CenterPadding(vit.patch_size)(frame).cuda()
    assert x.shape == (1, 3, 490, 854)
    with torch.no_grad():
        got = m(x)
        torch.cuda.synchronize()
        assert got.shape == (1, 120, 211, C)
        dev = lambda d: {k: v.cuda() for k, v in d.items()}  # noqa: E731
        feats = OV.forward_intermediates(dev(vsd), cfg, x, [cfg.depth - 1], stride=4)[0]
        ref = OD.forward(dev(sd), feats.permute(0, 2, 3, 1), hw)
    assert _lib.device_error() == 0
    mc = _min_cos(got, ref)
    assert mc > 0.999, f"stride-4 denoised backbone: min per-patch cosine {mc}"
