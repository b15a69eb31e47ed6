"""torch-autograd checker of the Swin-T training step (modules/swin_transformer.py:62-80, :234-325, :419-518 in train mode, then
modules/yolact.py's FPN / ProtoNet / heads and the four losses): the Swin counterpart of oracle/train_torch.forward_train, with the
same `taps` / `act` / `subst` mechanism and the stochastic-depth masks passed in (the engine draws them on the device; tests hand
its draws to this checker through TrainEngine.read_output('drop_path')).

Tensor names are the engine's (include/yolact_b200.h, yb_train_read); taps hold NCHW views of the [B, H*W, C] token tensors."""
import torch
import torch.nn.functional as F

from oracle import forward_torch as ft, train_torch as tt

DROP_PATH_RATE = 0.2


def drop_rates():
    """modules/swin_transformer.py:464: one rate per block over the four stages."""
    return [x.item() for x in torch.linspace(0, DROP_PATH_RATE, sum(ft.SWIN_DEPTHS))]


def swin_backbone_train(net, img, q, tap, masks):
    """c3, c4, c5 (NCHW) of the Swin-T backbone in train mode.  masks: [B, 12, 2] 0/1 (block, attention | MLP branch)."""
    P = dict(net.named_parameters())
    B, _, S, _ = img.shape
    img = F.pad(img, (0, (4 - S % 4) % 4, 0, (4 - S % 4) % 4))
    ws, H = ft.SWIN_WS, (S + 3) // 4

    def tok(name, t, H):                                      # taps / substitution on the NCHW view of a token tensor
        C = t.shape[-1]
        return tap(name, t.transpose(1, 2).reshape(B, C, H, H)).flatten(2).transpose(1, 2)
    lin = lambda t, p, bias=True: F.linear(t, q(P[p + '.weight']), P[p + '.bias'] if bias else None)
    x = F.conv2d(img, P['backbone.patch_embed.proj.weight'], P['backbone.patch_embed.proj.bias'], stride=4)       # fp32, as the engine
    x = tok('patch_embed', q(ft._ln(x.flatten(2).transpose(1, 2), P, 'backbone.patch_embed.norm')), H)
    rates, blk, feats = drop_rates(), 0, []
    for s, depth in enumerate(ft.SWIN_DEPTHS):
        heads, Hp = ft.SWIN_HEADS[s], -(-H // ws) * ws
        mask = ft._shift_mask(Hp, Hp, ws, ws // 2).to(img.device)
        rel = ft._rel_index(ws).view(-1).to(img.device)
        for b in range(depth):
            p, shift, C = f'backbone.layers.{s}.blocks.{b}', ws // 2 if b % 2 else 0, x.shape[-1]
            h = tok(p + '.norm1', q(ft._ln(x, P, p + '.norm1')), H)
            qkv_tok = tok(p + '.attn.qkv', q(lin(h, p + '.attn.qkv')), H)
            padded = P[p + '.attn.qkv.bias'].view(1, 1, 1, -1).expand(B, Hp, Hp, 3 * C).clone()     # padding tokens: qkv == bias
            padded[:, :H, :H] = qkv_tok.view(B, H, H, 3 * C)
            if shift:
                padded = torch.roll(padded, shifts=(-shift, -shift), dims=(1, 2))
            win = padded.view(B, Hp // ws, ws, Hp // ws, ws, 3 * C).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws * ws, 3 * C)
            B_, N = win.shape[0], ws * ws
            qkv = win.reshape(B_, N, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
            attn = (qkv[0] * (C // heads) ** -0.5) @ qkv[1].transpose(-2, -1)
            attn = attn + P[p + '.attn.relative_position_bias_table'][rel].view(N, N, -1).permute(2, 0, 1).unsqueeze(0)
            if shift:
                nW = mask.shape[0]
                attn = (attn.view(B_ // nW, nW, heads, N, N) + mask.unsqueeze(1).unsqueeze(0)).view(-1, heads, N, N)
            o = (attn.softmax(-1) @ qkv[2]).transpose(1, 2).reshape(B_, N, C)
            o = o.view(B, Hp // ws, Hp // ws, ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(B, Hp, Hp, C)
            if shift:
                o = torch.roll(o, shifts=(shift, shift), dims=(1, 2))
            o = tok(p + '.attn', q(o[:, :H, :H, :].reshape(B, H * H, C)), H)
            keep = 1 - rates[blk]
            dp = lambda t, br: t if rates[blk] == 0 else t.div(keep) * masks[:, blk, br].view(B, 1, 1)   # DropPath.forward (:68-80)
            x = tok(p + '.x1', q(x + dp(tok(p + '.attn.proj', q(lin(o, p + '.attn.proj')), H), 0)), H)
            m = tok(p + '.mlp.fc1', q(lin(tok(p + '.norm2', q(ft._ln(x, P, p + '.norm2')), H), p + '.mlp.fc1')), H)
            m = tok(p + '.mlp.fc2', q(lin(tok(p + '.mlp.gelu', q(F.gelu(m)), H), p + '.mlp.fc2')), H)
            x = tok(p + '.out', q(x + dp(m, 1)), H)
            blk += 1
        if s > 0:
            feats.append(tok(f'c{s + 2}', q(ft._ln(x, P, f'backbone.norm{s}')), H).transpose(1, 2).reshape(B, -1, H, H))
        if s < 3:
            p, C, Hn = f'backbone.layers.{s}.downsample', x.shape[-1], (H + 1) // 2
            g = F.pad(x.view(B, H, H, C), (0, 0, 0, H % 2, 0, H % 2))
            g = tok(p + '.merge', torch.cat([g[:, 0::2, 0::2], g[:, 1::2, 0::2], g[:, 0::2, 1::2], g[:, 1::2, 1::2]], -1).view(B, -1, 4 * C), Hn)
            x = tok(p + '.reduction', q(lin(tok(p + '.norm', q(ft._ln(g, P, p + '.norm')), Hn), p + '.reduction', bias=False)), Hn)
            H = Hn
    return feats


def forward_train(net, img, masks, taps=None, act=None, subst=None):
    """oracle/train_torch.forward_train for the Swin-T backbone (same taps / act / subst semantics)."""
    q = (lambda t: t) if act is None else (lambda t: t.to(act).float())

    def tap(name, t):
        if subst is not None:
            v = subst(name)
            if v is not None:
                t = v.to(t.dtype) + (t - t.detach())
        if taps is not None:
            if t.requires_grad:
                t.retain_grad()
            taps[name] = t
        return t
    c3, c4, c5 = swin_backbone_train(net, img, q, tap, masks)
    # FPN / ProtoNet / heads: as oracle/train_torch.forward_train after its backbone
    fpn, _conv = net.fpn, tt._conv
    up = lambda t, like: F.interpolate(t, size=like.shape[2:], mode='bilinear', align_corners=False)
    p5_1 = q(_conv(fpn.lat_layers[2], c5, q))
    l4 = q(_conv(fpn.lat_layers[1], c4, q))
    p4_1 = q(l4 + up(p5_1, l4))
    l3 = q(_conv(fpn.lat_layers[0], c3, q))
    p3_1 = q(l3 + up(p4_1, l3))
    tap('p5_1', p5_1); tap('p4_1', p4_1); tap('p3_1', p3_1)
    cr = lambda seq, t: q(F.relu(_conv(seq[0], t, q)))
    p5, p4, p3 = tap('p5', cr(fpn.pred_layers[2], p5_1)), tap('p4', cr(fpn.pred_layers[1], p4_1)), tap('p3', cr(fpn.pred_layers[0], p3_1))
    p6 = tap('p6', cr(fpn.downsample_layers[0], p5))
    p7 = tap('p7', cr(fpn.downsample_layers[1], p6))
    pn = net.proto_net
    t = p3
    for i in (0, 2, 4):
        t = tap(f'proto1.{i}', q(F.relu(_conv(pn.proto1[i], t, q))))
    t = tap('proto.up', q(F.interpolate(t, scale_factor=2, mode='bilinear', align_corners=True)))
    t = tap('proto2.0', q(F.relu(_conv(pn.proto2[0], t, q))))
    proto = F.relu(_conv(pn.proto2[2], t, q)).permute(0, 2, 3, 1).contiguous()
    pl, B = net.prediction_layers, img.shape[0]
    cls, box, coef = [], [], []
    for li, lv in enumerate((p3, p4, p5, p6, p7)):
        f = tap(f'head.f{li}', q(F.relu(_conv(pl.upfeature[0], lv, q))))
        cls.append(_conv(pl.conf_layer, f, q).permute(0, 2, 3, 1).reshape(B, -1, pl.num_classes))
        box.append(_conv(pl.bbox_layer, f, q).permute(0, 2, 3, 1).reshape(B, -1, 4))
        coef.append(torch.tanh(_conv(pl.coef_layer[0], f, q)).permute(0, 2, 3, 1).reshape(B, -1, pl.coef_dim))
    seg = _conv(net.semantic_seg_conv, p3, q)
    return (tap('out.cls', torch.cat(cls, 1)), tap('out.box', torch.cat(box, 1)), tap('out.coef', torch.cat(coef, 1)), tap('out.proto', proto),
            tap('out.seg', seg))


def training_step_forward(net, img, box_classes, masks_gt, drop_masks, taps=None, act=None, subst=None):
    """The reference's four losses of a Swin-T training step with the given stochastic-depth masks."""
    return tt.compute_loss(net, *forward_train(net, img, drop_masks, taps, act, subst), box_classes, masks_gt)
