"""Training conformance of stages 2 and 3: every gradient of the CUDA training step against the fp64 mirror of
tests/train_oracle_fp64.py, per element, node by node and end to end.

One real training step per case (`PretrainedViTWrapper` in training mode, or `Denoiser`, then `denoise_loss` and
backward).  Recorders around the train_ops entry points keep each node's output, saved tensors and the gradient that
reaches it.  Then:
  * node level, teacher-forced: each node's saved activations against fp64 of their ops (forward conformance), and every
    gradient the node returned against the mirror fed the node's own incoming gradient;
  * model level: the mirror chained from the loss back to the parameters, the incoming-gradient variance carried from
    node to node, and the glue (pos_embed slicing and resampling, cls + pos, register rows, the Denoiser's PE)
    re-evaluated in fp64.  Every parameter is checked, including cls_token, reg_token, pos_embed, every ls*.gamma, every
    bias and norm_pre.
Each case runs in default mode and under torch.use_deterministic_algorithms(True) (other kernels: attention_bwd_det,
wgrad_ordered, colsum_ordered, denoise_loss_ordered, _ResampleFn); the DINOv2 and SwiGLU cases also with gradient
checkpointing, whose deterministic gradients must equal the stored-activation run bit for bit."""
import re

import pytest
import torch

import train_oracle_fp64 as T
import vit_oracle_rope as R

pytestmark = pytest.mark.gpu

BLOCK_NAMES = {"n1w": "norm1.weight", "n1b": "norm1.bias", "wq": "attn.qkv.weight", "qkvb": "attn.qkv.bias",
               "wp": "attn.proj.weight", "projb": "attn.proj.bias", "ls1": "ls1.gamma", "n2w": "norm2.weight",
               "n2b": "norm2.bias", "w1": "mlp.fc1.weight", "fc1b": "mlp.fc1.bias", "w2": "mlp.fc2.weight",
               "fc2b": "mlp.fc2.bias", "ls2": "ls2.gamma"}

# Tokens per image (ntok) against the attention backward's 128-key tiles (one CTA per key tile; dQ of several tiles is
# reduced across CTAs in default mode and looped over in attention_bwd_det), B * ntok against the 64- / 128-row GEMM tiles,
# and the split-K factor of `wgrad` (train_ops.wgrad_splits: 2 once the rows reach 8 k-blocks of 64) -- asserted by
# test_cases_cross_the_tile_and_split_boundaries.
VIT_CASES = {
    # 61 tokens (one key tile), 122 rows, pos resampled 7x7 -> 7x8, unsplit wgrad
    "dinov2-s14-reg4": dict(ident="vit_small_patch14_reg4_dinov2.lvd142m", stride=14, depth=2, img=98, B=2, hw=(98, 112),
                            ckpt=True),
    # 86 tokens, 258 rows (a ragged 64-row tile), unsplit wgrad
    "dinov2-s14-reg4-stride7": dict(ident="vit_small_patch14_reg4_dinov2.lvd142m", stride=7, depth=2, img=98, B=3,
                                    hw=(70, 70), ckpt=True),
    # 174 tokens: two key tiles, the second ragged (46 keys); 522 rows: split-K wgrad (2 splits) on every layer
    "dinov2-s14-reg4-stride7-174tok": dict(ident="vit_small_patch14_reg4_dinov2.lvd142m", stride=7, depth=2, img=98, B=3,
                                           hw=(98, 98), ckpt=True),
    # 43 tokens, 129 rows (one row past two 64-row tiles), no LayerScale
    "dino-s16-resampled": dict(ident="vit_small_patch16_224.dino", stride=16, depth=2, img=None, B=3, hw=(96, 112),
                               ckpt=False),
    # 21 tokens, batch 1: pre-norm, no patch bias
    "clip-b16": dict(ident="vit_base_patch16_clip_224.openai", stride=16, depth=2, img=64, B=1, hw=(64, 80), ckpt=False),
    # 21 tokens, 42 rows: head_dim 80
    "mae-h14": dict(ident="vit_huge_patch14_224.mae", stride=14, depth=1, img=56, B=2, hw=(56, 70), ckpt=False),
    # 29 tokens, 87 rows: SwiGLU
    "vitg-swiglu": dict(ident="vit_giant_patch14_dinov2.lvd142m", stride=14, depth=1, img=56, B=3, hw=(56, 98), ckpt=True),
    # 29 tokens, 87 rows: RoPE with 5 prefix rows
    "dinov3-s16": dict(ident="vit_small_patch16_dinov3.lvd1689m", stride=16, depth=2, img=None, B=3, hw=(64, 96),
                       ckpt=False),
}
DEN_CASES = {
    # 156 tokens: two key tiles, the second ragged (28 keys); 468 rows: split-K wgrad (2 splits); PE resampled 5x6 -> 12x13
    "denoiser-1blk": dict(blocks=1, C=384, noise=(5, 6), B=3, hw=(12, 13)),
    # 72 tokens, 144 rows, unsplit wgrad; PE resampled 8x8 -> 9x8
    "denoiser-2blk": dict(blocks=2, C=384, noise=(8, 8), B=2, hw=(9, 8)),
}


def _dev_ok():
    from dvt import _lib
    torch.cuda.synchronize()
    assert _lib.device_error() == 0


# ------------------------------------------------------------------------------------------------ recording
class Recorder:
    """Wraps the train_ops node entry points: keeps (kind, output, node info) per call and the gradient reaching each
    output and each glue tensor."""

    def __init__(self, monkeypatch):
        from dvt import train_ops
        self.nodes = []
        self.grads = {}
        orig = {k: getattr(train_ops, k) for k in ("vit_embed", "vit_layernorm", "vit_block_forward", "vit_norm_strip",
                                                   "block_forward")}

        def hook(key):
            def f(g):
                self.grads[key] = g.detach().clone()
            return f

        def wrap(kind):
            def f(*a, **k):
                y = orig[kind](*a, **k)
                i = len(self.nodes)
                info = {"args": a, "kw": k, "fn": y.grad_fn}
                if kind in ("vit_block_forward", "block_forward"):
                    info["saved"] = [None if t is None else t.detach().clone() for t in y.grad_fn.saved_tensors]
                    info["x0"] = a[0].detach().clone()
                elif kind in ("vit_layernorm", "vit_norm_strip"):
                    info["x0"] = a[0].detach().clone()
                elif kind == "vit_embed":
                    info["patches"] = y.grad_fn.saved_tensors[0].detach().clone()
                    for j, nm in ((3, "pos"), (4, "prefix")):
                        if a[j] is not None and a[j].requires_grad:
                            a[j].register_hook(hook((i, nm)))
                if kind != "vit_embed":
                    a[0].register_hook(hook((i, "in")))
                y.register_hook(hook((i, "out")))
                self.nodes.append((kind, y, info))
                return y
            return f

        for k in orig:
            monkeypatch.setattr(train_ops, k, wrap(k))


def _block_wts(kind, info, blk):
    """The prepared weights the node ran with, as a dict of BLOCK_WTS."""
    if kind == "vit_block_forward":
        return dict(zip(T.BLOCK_WTS, info["fn"].wts))
    s = info["saved"]
    f32 = lambda t: t.detach().float()             # noqa: E731
    return dict(n1w=s[13], n1b=f32(blk.norm1.bias), wq=s[9], qkvb=f32(blk.attn.qkv.bias), wp=s[10],
                projb=f32(blk.attn.proj.bias), ls1=None, n2w=s[14], n2b=f32(blk.norm2.bias), w1=s[11],
                fc1b=f32(blk.mlp.fc1.bias), w2=s[12], fc2b=f32(blk.mlp.fc2.bias), ls2=None)


def _block_acts(kind, info, wts, heads, batch, eps, rope):
    from dvt import train_ops
    s = info["saved"]
    if kind == "block_forward":
        x1, xn1, qkv, att, lse, xn2, hpre, hid = s[1:9]
        return dict(x1=x1, xn1=xn1, qkv=qkv, att=att, lse=lse, br1=None, xn2=xn2, hpre=hpre, hid=hid, br2=None)
    if info["fn"].checkpoint:     # the backward recomputes them with the same kernels: the same bits
        _, acts = train_ops._vit_block_fwd(s[0], tuple(wts[k] for k in T.BLOCK_WTS), heads, batch, keep=True, eps=eps,
                                           rope=rope)
        return dict(zip(T.BLOCK_ACTS, acts))
    return dict(zip(T.BLOCK_ACTS, s[1:]))


# ------------------------------------------------------------------------------------------------ checking
class Report:
    def __init__(self, case):
        self.case, self.rows, self.bad = case, [], []

    def grad(self, what, got, ref: T.G):
        worst, rms = T.ratio(got, ref)
        self.rows.append(f"  {what:<40s} worst {worst:6.3f}  rms {rms:6.3f}")
        if not worst <= 1.0:
            self.bad.append(f"{what}: worst ratio {worst:.3g}")

    def fwd(self, what, ratios):
        w = max(ratios.values())
        self.rows.append(f"  {what:<40s} forward worst {w:6.3f}")
        if not w <= 1.0:
            self.bad.append(f"{what} forward: {ratios}")

    def done(self):
        print(f"\n[{self.case}]\n" + "\n".join(self.rows))
        assert not self.bad, f"{self.case}: " + "; ".join(self.bad)


def _prepared_weights_are_the_modules(kind, wts, blk):
    """The weights a block node ran with are the casts of the module's current parameters: bf16 GEMM weights, fp32
    LayerNorm / bias / LayerScale (a stale or wrong weight preparation would otherwise be mirrored faithfully)."""
    b16 = lambda t: t.detach().to(torch.bfloat16)          # noqa: E731
    f32 = lambda t: t.detach().float()                     # noqa: E731
    want = {"wq": b16(blk.attn.qkv.weight), "wp": b16(blk.attn.proj.weight), "w1": b16(blk.mlp.fc1.weight),
            "w2": b16(blk.mlp.fc2.weight), "n1w": f32(blk.norm1.weight), "n2w": f32(blk.norm2.weight)}
    if kind == "vit_block_forward":
        want.update(n1b=f32(blk.norm1.bias), qkvb=f32(blk.attn.qkv.bias), projb=f32(blk.attn.proj.bias),
                    n2b=f32(blk.norm2.bias), fc1b=f32(blk.mlp.fc1.bias), fc2b=f32(blk.mlp.fc2.bias),
                    ls1=f32(blk.ls1.gamma) if hasattr(blk.ls1, "gamma") else None,
                    ls2=f32(blk.ls2.gamma) if hasattr(blk.ls2, "gamma") else None)
    for k, v in want.items():
        assert (v is None) == (wts[k] is None) and (v is None or torch.equal(wts[k], v)), f"prepared weight {k} is stale"


def _check(rec, model_params, blocks, heads, report, *, eps, glue, blk_prefix=lambda i: f"blocks.{i}.", rope_expect=None):
    """Node-level and model-level checks of one recorded step.  glue(dprefix G, dpos G) -> {param name: G} re-evaluates
    the position / prefix glue in fp64 (model level).  eps is the architecture's LayerNorm eps and rope_expect the
    (table, prefix) its blocks must run with (None: no RoPE); both are asserted, not taken from the nodes.  Returns the
    chained gradient of the first node's input."""
    nodes = rec.nodes
    g_chain = None
    blk_i = len(blocks) - 1
    for i in reversed(range(len(nodes))):
        kind, y, info = nodes[i]
        g_in = rec.grads[(i, "out")]
        if g_chain is None:   # the last node: its incoming gradient is the loss gradient
            pred, target = rec.loss_args
            g_chain = T.loss_bwd(pred, target)
            report.grad("loss dpred", g_in.reshape(g_chain.val.shape), g_chain)
            g_chain = g_chain.reshape(g_in.shape)
        if kind in ("vit_block_forward", "block_forward"):
            blk = blocks[blk_i]
            fn = info["fn"]
            batch = fn.batch if kind == "vit_block_forward" else info["args"][3]
            rope = fn.rope if kind == "vit_block_forward" else None
            beps = fn.eps if kind == "vit_block_forward" else 1e-6
            assert beps == eps, (beps, eps)
            if rope_expect is None:
                assert rope is None
            else:
                assert rope[1] == rope_expect[1], "RoPE prefix"
                assert torch.allclose(rope[0].cpu(), rope_expect[0], rtol=0, atol=1e-6), "RoPE table of another grid"
            wts = _block_wts(kind, info, blk)
            _prepared_weights_are_the_modules(kind, wts, blk)
            acts = _block_acts(kind, info, wts, heads, batch, beps, rope)
            report.fwd(f"{blk_prefix(blk_i)}saved tensors", T.check_block_forward(info["x0"], acts, wts, y.detach(), heads=heads,
                                                                              batch=batch, eps=beps, rope=rope))
            node = T.block_bwd(info["x0"], acts, wts, T.exact(g_in), heads=heads, batch=batch, eps=beps, rope=rope)
            chain = T.block_bwd(info["x0"], acts, wts, g_chain, heads=heads, batch=batch, eps=beps, rope=rope)
            for k, nm in BLOCK_NAMES.items():
                if k in node:
                    p = getattr_path(blk, nm)
                    report.grad(f"node  {blk_prefix(blk_i)}{nm}", p.grad.reshape(node[k].val.shape), node[k])
                    report.grad(f"model {blk_prefix(blk_i)}{nm}", p.grad.reshape(chain[k].val.shape), chain[k])
            report.grad(f"node  {blk_prefix(blk_i)}dx0", rec.grads[(i, "in")], node["x0"])
            g_chain = chain["x0"]
            blk_i -= 1
        elif kind in ("vit_layernorm", "vit_norm_strip"):
            x, w_, b_ = info["x0"], info["args"][1], info["args"][2]
            assert info["args"][-1 if kind == "vit_layernorm" else 5] == eps
            if kind == "vit_layernorm":
                report.fwd("norm_pre output", {"y": T.ln_excess(y, x, w_, b_, eps)})
                node = T.layernorm_bwd(x, w_.detach(), T.exact(g_in), eps)
                chain = T.layernorm_bwd(x, w_.detach(), g_chain, eps)
                label = "norm_pre"
            else:
                ntok, prefix = info["args"][3], info["args"][4]
                C_ = x.shape[1]
                kept = x.view(-1, ntok, C_)[:, prefix:].reshape(-1, C_)
                report.fwd("norm output", {"y": T.ln_excess(y, kept, w_, b_, eps)})
                g2 = g_in.reshape(-1, x.shape[1])
                node = T.norm_strip_bwd(x, w_.detach(), T.exact(g2), ntok=ntok, prefix=prefix, eps=eps)
                chain = T.norm_strip_bwd(x, w_.detach(), g_chain.reshape(-1, x.shape[1]), ntok=ntok, prefix=prefix, eps=eps)
                label = "norm"
            for k, nm, p in (("w", "weight", w_), ("b", "bias", b_)):
                report.grad(f"node  {label}.{nm}", p.grad, node[k])
                report.grad(f"model {label}.{nm}", p.grad, chain[k])
            report.grad(f"node  {label} dx", rec.grads[(i, "in")], node["x"])
            g_chain = chain["x"]
        elif kind == "vit_embed":
            C, _, P, _ = info["args"][1].shape
            batch, prefix = info["fn"].meta[0], info["fn"].meta[1]
            node = T.embed_bwd(info["patches"], T.exact(g_in), batch=batch, prefix=prefix, C=C, P=P)
            chain = T.embed_bwd(info["patches"], g_chain, batch=batch, prefix=prefix, C=C, P=P)
            pw, pb = info["args"][1], info["args"][2]
            report.fwd("patch embedding output", T.check_embed_forward(y, info["patches"], pw, pb, info["args"][3],
                                                                       info["args"][4], batch=batch))
            report.grad("node  patch_embed.proj.weight", pw.grad, node["pe_w"])
            report.grad("model patch_embed.proj.weight", pw.grad, chain["pe_w"])
            if pb is not None:
                report.grad("node  patch_embed.proj.bias", pb.grad, node["pe_b"])
                report.grad("model patch_embed.proj.bias", pb.grad, chain["pe_b"])
            if (i, "pos") in rec.grads:
                report.grad("node  dpos", rec.grads[(i, "pos")], node["pos"])
            report.grad("node  dprefix", rec.grads[(i, "prefix")], node["prefix"])
            for nm, ref in glue(chain["prefix"], chain["pos"] if info["args"][3] is not None else None).items():
                report.grad(f"model {nm}", model_params[nm].grad.reshape(ref.val.shape), ref)
            g_chain = None
    return g_chain


def getattr_path(m, path):
    for p in path.split("."):
        m = getattr(m, p)
    return m


# ------------------------------------------------------------------------------------------------ stage 3
def _vit(case, seed=3):
    import dvt.models as DVT
    from dvt.models import vit_wrapper as VW
    from oracle import vit as OV
    c = VIT_CASES[case]
    a = dict(VW.arch_of(c["ident"]), depth=c["depth"])
    if c["img"]:
        a["img"] = c["img"]
    P = int(re.search(r"patch(\d+)", c["ident"]).group(1))
    if a["rope"]:
        cfg = R.RopeViTConfig(a["embed"], a["depth"], a["heads"], P, a["img"], a["mlp"], num_reg_tokens=a["reg"],
                              no_embed_class=True, ln_eps=a["ln_eps"])
        sd = R.random_state_dict(cfg, seed=seed)
    else:
        cfg = OV.ViTConfig(a["embed"], a["depth"], a["heads"], P, a["img"], a["mlp"], a["swiglu"], a["ls"], a["reg"],
                           a["no_embed_class"], a["ln_eps"])
        sd = OV.random_state_dict(cfg, seed=seed)
        if not a["patch_bias"]:
            del sd["patch_embed.proj.bias"]
        if a["pre_norm"]:
            g = torch.Generator().manual_seed(seed + 1)
            sd["norm_pre.weight"] = 1 + 0.1 * torch.randn(a["embed"], generator=g)
            sd["norm_pre.bias"] = 0.1 * torch.randn(a["embed"], generator=g)
    w = DVT.PretrainedViTWrapper(c["ident"], stride=c["stride"], allow_random_init=True)
    w.model = VW.B200VisionTransformer(c["ident"], P, a)
    w.model.patch_embed.proj.stride = [c["stride"], c["stride"]]
    w.model.load_state_dict(sd, strict=True)
    return w.cuda(), a, P


def _vit_step(monkeypatch, w, x, target, ckpt):
    from dvt import train_ops
    with monkeypatch.context() as mp:
        rec = Recorder(mp)
        w.set_trainable(True)
        w.model.set_grad_checkpointing(ckpt)
        for p in w.parameters():
            p.grad = None
        pred = w.get_intermediate_layers(x)[0].permute(0, 2, 3, 1)
        rec.loss_args = (pred.detach().clone(), target)
        loss, _, _ = train_ops.denoise_loss(pred, target)
        loss.backward()
    _dev_ok()
    return rec


def _vit_glue(m, a, hw_tok):
    """Model-level glue: (dprefix, dpos) of the embedding node -> gradients of cls_token, reg_token and pos_embed.  The
    values come from fp64 autograd through oracle/vit.py's restatement of timm `_pos_embed` (resample_abs_pos_embed,
    cls + pos[0] unless no_embed_class, register rows), not from the wrapper's `_pos_tables_train`, so a misreading shared
    by the wrapper and this test would still show.  The variances come from the mirror's linear pass (the resample
    transpose on squared weights)."""
    from oracle import vit as OV

    def glue(dprefix: T.G, dpos):
        dev = dprefix.val.device
        names = [k for k in ("cls_token", "reg_token", "pos_embed") if hasattr(m, k)]
        leaves = {k: getattr(m, k).detach().double().cpu().requires_grad_(True) for k in names}
        npre = 0 if a["no_embed_class"] else 1
        rows, outs, gouts = [leaves["cls_token"][0]], [], []
        if dpos is not None:
            pos = OV.resample_abs_pos_embed(leaves["pos_embed"], hw_tok, m.native_grid, npre)
            outs.append(pos[0, npre:])
            gouts.append(dpos.val.cpu())
            if npre:
                rows = [rows[0] + pos[0, :1]]
        if a["reg"]:
            rows.append(leaves["reg_token"][0])
        outs.append(torch.cat(rows))
        gouts.append(dprefix.val.cpu())
        val = dict(zip(names, torch.autograd.grad(outs, [leaves[k] for k in names], gouts, allow_unused=True)))
        var = {"cls_token": dprefix.var[0:1]}
        if a["reg"]:
            var["reg_token"] = dprefix.var[1:1 + a["reg"]]
        if dpos is not None:
            h, w = hw_tok
            gh, gw = m.native_grid
            C = dpos.val.shape[1]
            pv = dpos.var
            if (h, w) != (gh, gw):
                d = T.resample_bwd(T.G(dpos.val.t().reshape(1, C, h, w), dpos.var.t().reshape(1, C, h, w)), gh, gw)
                pv = d.var[0].reshape(C, -1).t()
            var["pos_embed"] = pv if a["no_embed_class"] else torch.cat([dprefix.var[0:1], pv])
        return {k: T.G(val[k].to(dev).reshape(v.shape), v) for k, v in var.items()}
    return glue


def _vit_run(case, det, ckpt, monkeypatch):
    c = VIT_CASES[case]
    w, a, P = _vit(case)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(c["B"], 3, *c["hw"], generator=g).cuda()
    h, wd = (c["hw"][0] - P) // c["stride"] + 1, (c["hw"][1] - P) // c["stride"] + 1
    target = torch.randn(c["B"], h, wd, a["embed"], generator=g).cuda()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        rec = _vit_step(monkeypatch, w, x, target, ckpt)
    finally:
        torch.use_deterministic_algorithms(prev)
    return w, a, rec, (h, wd)


@pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])
@pytest.mark.parametrize("case", list(VIT_CASES))
def test_vit_training_step_matches_fp64_mirror(case, det, monkeypatch):
    c = VIT_CASES[case]
    variants = [False, True] if c["ckpt"] else [False]
    grads = []
    for ckpt in variants:
        w, a, rec, hw_tok = _vit_run(case, det, ckpt, monkeypatch)
        params = dict(w.model.named_parameters())
        report = Report(f"{case} {'det' if det else 'default'}{' ckpt' if ckpt else ''}")
        rope = None
        if a["rope"]:
            cos, sin = R.rope_cos_sin(*hw_tok)
            rope = (torch.cat([cos[:, :32], sin[:, :32]], 1), 1 + a["reg"])
        _check(rec, params, list(w.model.blocks), a["heads"], report, eps=a["ln_eps"], glue=_vit_glue(w.model, a, hw_tok),
               rope_expect=rope)
        missing = [k for k in params if not any(r.split()[:2] == ["model", k] for r in report.rows)]
        assert not missing, missing                  # every parameter was checked
        report.done()
        grads.append({k: p.grad.detach().clone() for k, p in params.items()})
        _dev_ok()
    if det and len(grads) == 2:
        for k in grads[0]:
            assert torch.equal(grads[0][k], grads[1][k]), f"{case}: checkpointed gradient of {k} differs"


# ------------------------------------------------------------------------------------------------ stage 2
@pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])
@pytest.mark.parametrize("case", list(DEN_CASES))
def test_denoiser_training_step_matches_fp64_mirror(case, det, monkeypatch):
    import dvt.models as DVT
    from dvt import train_ops
    from oracle import denoiser as OD
    from oracle import vit as OV
    OD_resample = lambda pos, hw, noise: OV.resample_abs_pos_embed(pos, hw, noise, 0)   # noqa: E731
    c = DEN_CASES[case]
    den = DVT.Denoiser(*c["noise"], c["C"], vit=None, num_blocks=c["blocks"])
    den.load_state_dict(OD.random_state_dict(c["C"], c["noise"], c["blocks"], seed=5), strict=True)
    den = den.cuda()
    g = torch.Generator().manual_seed(6)
    x = torch.randn(c["B"], *c["hw"], c["C"], generator=g).cuda()
    target = torch.randn(c["B"], *c["hw"], c["C"], generator=g).cuda()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        with monkeypatch.context() as mp:
            rec = Recorder(mp)
            pred = den(x)
            rec.loss_args = (pred.detach().clone(), target)
            loss, _, _ = train_ops.denoise_loss(pred, target)
            loss.backward()
    finally:
        torch.use_deterministic_algorithms(prev)
    _dev_ok()
    report = Report(f"{case} {'det' if det else 'default'}")
    pre = (lambda i: "denoiser.") if c["blocks"] == 1 else (lambda i: f"denoiser.{i}.")
    g_chain = _check(rec, {}, den._blocks(), c["C"] // 64, report, eps=1e-6, glue=None, blk_prefix=pre)
    # the Denoiser's PE: t = x + resample(pos_embed), summed over the batch, then the resample transpose
    B, (h, w), C = c["B"], c["hw"], c["C"]
    d = g_chain.reshape(B, h * w, C)
    d = T.G(d.val.sum(0), d.var.sum(0) + B * (T.U_32 * d.val.abs().sum(0)) ** 2)
    d = T.G(d.val.t().reshape(1, C, h, w), d.var.t().reshape(1, C, h, w))
    var = T.resample_bwd(d, *c["noise"]).var[0].reshape(C, -1).t()
    # the value by fp64 autograd through oracle/denoiser.py's PE (resample_abs_pos_embed, no prefix)
    pos = den.pos_embed.detach().double().cpu().requires_grad_(True)
    (val,) = torch.autograd.grad(OD_resample(pos, (h, w), c["noise"]), pos, d.val[0].reshape(C, -1).t()[None].cpu())
    report.grad("model pos_embed", den.pos_embed.grad[0], T.G(val[0].to(var.device), var))
    missing = [k for k, _ in den.named_parameters() if not any(r.split()[:2] == ["model", k] for r in report.rows)]
    assert not missing, missing                      # every parameter was checked
    report.done()


def test_cases_cross_the_tile_and_split_boundaries():
    """The configurations above reach what real shapes (257, 1025 tokens) take: several key tiles with a ragged last one,
    in both stages, and split-K weight gradients; and also the single-tile, unsplit forms."""
    from dvt import train_ops
    vit, den = [], []
    for c in VIT_CASES.values():
        P = int(re.search(r"patch(\d+)", c["ident"]).group(1))
        h, w = ((n - P) // c["stride"] + 1 for n in c["hw"])
        reg = 4 if ("reg4" in c["ident"] or "dinov3" in c["ident"]) else 0
        vit.append((1 + reg + h * w, c["B"]))
    den = [(c["hw"][0] * c["hw"][1], c["B"]) for c in DEN_CASES.values()]
    for cases in (vit, den):
        assert any(n > 128 and n % 128 for n, _ in cases)           # several key tiles, the last ragged
        assert any(n <= 128 for n, _ in cases)                      # one key tile
        splits = [train_ops.wgrad_splits(n * b, 384, 384) for n, b in cases]
        assert max(splits) >= 2 and min(splits) == 1, splits
    assert any(b % 2 for _, b in vit + den)
