"""Synthetic weights / inputs of the benchmark workloads (SURVEY.md section 8d): there is no network
access for checkpoints or datasets, so bench.py and the tests use random-init weights of the reference
architecture and Cityscapes-/COCO-shaped random images."""
import numpy as np
import torch


def synthetic_model(cfg=None, depth=(3, 4, 6, 3), seed=0, device="cpu"):
    """Random-init resnet_upsnet per SURVEY.md section 8d config 2: reference initialisers, except
    (a) offset convs get non-zero weights/biases so DCN offsets are a few pixels (the reference zero-inits
    them, modules/deform_conv.py:72-73 -- zero offsets would hide DCN bugs), (b) BN statistics are
    randomised so folding is exercised, (c) the class / mask heads are biased so that several dozen
    detections survive score > 0.6 and reach the panoptic head, (d) GroupNorm affines are randomised around (1, 0)."""
    from upsnet_b200.model import resnet_upsnet, Bottleneck
    from upsnet_b200.operators import DeformConvWithOffset
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad(), torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)          # module constructors draw from the global CPU generator
        m = resnet_upsnet(list(depth), cfg)
        for prm in m.parameters():       # DeformConv creates its parameters on CUDA (like the reference):
            if prm.is_cuda:              # re-draw them from the CPU generator so every build is identical
                prm.copy_(torch.empty(prm.shape).uniform_(-0.05, 0.05, generator=g).to(prm.device))
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.weight.copy_(torch.empty_like(mod.weight).uniform_(0.5, 1.5, generator=g))
                mod.bias.copy_(torch.empty_like(mod.bias).normal_(0, 0.1, generator=g))
                mod.running_mean.copy_(torch.empty_like(mod.running_mean).normal_(0, 0.1, generator=g))
                mod.running_var.copy_(torch.empty_like(mod.running_var).uniform_(0.5, 1.5, generator=g))
            elif isinstance(mod, DeformConvWithOffset):
                # offsets of a few pixels, like a trained DCN: a per-tap constant (bias ~ N(0,1.5 px)) plus a
                # small input-dependent part (FPN features are calibrated to RMS 1 below)
                w = mod.conv_offset.weight
                w.copy_(torch.empty(w.shape).normal_(0, 0.5 / (w.shape[1] * 9) ** 0.5, generator=g).to(w.device))
                mod.conv_offset.bias.copy_(torch.empty(mod.conv_offset.bias.shape).normal_(0, 1.5, generator=g))
                cw = mod.conv.weight
                cw.copy_(torch.empty(cw.shape).normal_(0, (2.0 / (cw.shape[1] * 9)) ** 0.5, generator=g).to(cw.device))
                mod.conv.bias.zero_()
            elif isinstance(mod, Bottleneck):
                for c in (mod.conv1, mod.conv2, mod.conv3):
                    w = c.weight
                    fan = w.shape[1] * w.shape[2] * w.shape[3]
                    w.copy_(torch.empty(w.shape).normal_(0, (2.0 / fan) ** 0.5, generator=g).to(w.device))
                if mod.deformable:
                    w = mod.conv2_offset.weight
                    w.copy_(torch.empty(w.shape).normal_(0, 0.01 / (w.shape[1] * 9) ** 0.5, generator=g))
                    mod.conv2_offset.bias.copy_(torch.empty(mod.conv2_offset.bias.shape).normal_(0, 1.5, generator=g))
                if mod.downsample is not None:
                    w = mod.downsample[0].weight
                    w.copy_(torch.empty(w.shape).normal_(0, (1.0 / w.shape[1]) ** 0.5, generator=g))
                mod.bn3.weight.mul_(0.3)  # keep the residual stream bounded at random init
        sw = m.resnet_backbone.conv1.conv1.weight
        sw.copy_(torch.empty(sw.shape).normal_(0, (2.0 / 147) ** 0.5 / 50, generator=g))
        # heads: make detections plentiful and confident enough for the panoptic branch
        m.rpn.cls_score.weight.copy_(torch.empty_like(m.rpn.cls_score.weight).normal_(0, 0.05, generator=g))
        m.rpn.bbox_pred.weight.copy_(torch.empty_like(m.rpn.bbox_pred.weight).normal_(0, 0.01, generator=g))
        m.rcnn.cls_score.weight.copy_(torch.empty_like(m.rcnn.cls_score.weight).normal_(0, 0.25, generator=g))
        m.rcnn.cls_score.bias[0] = -1.0
        m.rcnn.bbox_pred.weight.copy_(torch.empty_like(m.rcnn.bbox_pred.weight).normal_(0, 0.02, generator=g))
        m.mask_branch.mask_score.bias.fill_(0.2)
        m.fcn_head.score.weight.copy_(torch.empty_like(m.fcn_head.score.weight).normal_(0, 0.1, generator=g))
        for mod in m.modules():     # group_norm configurations: non-trivial affines (nn.GroupNorm inits 1 and 0)
            if isinstance(mod, torch.nn.GroupNorm):
                mod.weight.copy_(torch.empty_like(mod.weight).uniform_(0.5, 1.5, generator=g))
                mod.bias.copy_(torch.empty_like(mod.bias).normal_(0, 0.1, generator=g))
        if sum(depth) > 16:      # deeper than ResNet-50: keep the residual stream of the random-init stack bounded
            _calibrate_residual_growth(m, g)
        _calibrate_fpn_laterals(m, g)
    m = m.to(device)
    m.prepare()
    return m


def _calibrate_residual_growth(m, g):
    """A random-init residual stack multiplies its activation scale by ~1.8 per block; over the 23 blocks of a ResNet-101
    res4 stage that is 10^5 -- the DCN offset convs then ask for offsets of hundreds of pixels and the forward becomes
    chaotic (any two fp32 implementations diverge).  One torch-only pass over a small random image rescales every
    block's bn3 so that its residual branch has at most a quarter of the trunk's RMS (growth <= 3 % per block), like a
    trained network's.  ResNet-50 models are left exactly as in round 1."""
    import torch.nn.functional as F
    bb = m.resnet_backbone
    x = (torch.randn(1, 3, 96, 128, generator=g) * 50)
    cpu = lambda t: t.detach().float().cpu()   # noqa: E731

    def bn(t, b):
        return F.batch_norm(t, cpu(b.running_mean), cpu(b.running_var), cpu(b.weight), cpu(b.bias), False, 0.0, b.eps)

    t = F.max_pool2d(F.relu(bn(F.conv2d(x, cpu(bb.conv1.conv1.weight), None, 2, 3), bb.conv1.bn1)), 3, 2, 1)
    for blk in (bb.res2, bb.res3, bb.res4, bb.res5):
        for b in blk.layers:
            out = F.relu(bn(F.conv2d(t, cpu(b.conv1.weight), None, b.stride), b.bn1))
            out = F.relu(bn(F.conv2d(out, cpu(b.conv2.weight), None, 1, b.dilation, b.dilation), b.bn2))   # offsets ignored
            pre = F.conv2d(out, cpu(b.conv3.weight))
            branch = bn(pre, b.bn3)
            res = t if b.downsample is None else bn(F.conv2d(t, cpu(b.downsample[0].weight), None, b.stride), b.downsample[1])
            r_b, r_t = branch.pow(2).mean().sqrt().item(), res.pow(2).mean().sqrt().item()
            if r_b > 0.25 * r_t:
                s_ = 0.25 * r_t / r_b
                b.bn3.weight.mul_(s_); b.bn3.bias.mul_(s_)
                branch = bn(pre, b.bn3)
            t = F.relu(branch + res)


def _calibrate_fpn_laterals(m, g):
    """Random-init residual stacks let activation scale drift (C5 was ~50x C2), which saturates the
    softmax heads into exact ties and makes DCN offsets absurd.  One torch-only pass of the backbone over a
    small random image measures the RMS of every FPN lateral output and rescales that lateral conv to
    RMS 1, so P2..P6 -- and with them every head -- operate at O(1) like a trained network."""
    import torch.nn.functional as F
    bb = m.resnet_backbone
    x = (torch.randn(1, 3, 96, 128, generator=g) * 50)
    cpu = lambda t: t.detach().float().cpu()   # noqa: E731  (DeformConv parameters may live on CUDA)

    def bn(t, b):
        return F.batch_norm(t, cpu(b.running_mean), cpu(b.running_var), cpu(b.weight), cpu(b.bias), False, 0.0, b.eps)

    def bott(b, t):
        out = F.relu(bn(F.conv2d(t, cpu(b.conv1.weight), None, b.stride), b.bn1))
        out = F.relu(bn(F.conv2d(out, cpu(b.conv2.weight), None, 1, b.dilation, b.dilation), b.bn2))   # offsets ignored
        out = bn(F.conv2d(out, cpu(b.conv3.weight)), b.bn3)
        res = t if b.downsample is None else bn(F.conv2d(t, cpu(b.downsample[0].weight), None, b.stride), b.downsample[1])
        return F.relu(out + res)

    t = F.max_pool2d(F.relu(bn(F.conv2d(x, cpu(bb.conv1.conv1.weight), None, 2, 3), bb.conv1.bn1)), 3, 2, 1)
    feats = []
    for blk in (bb.res2, bb.res3, bb.res4, bb.res5):
        for b in blk.layers:
            t = bott(b, t)
        feats.append(t)
    for name, f in zip(("fpn_p2_1x1", "fpn_p3_1x1", "fpn_p4_1x1", "fpn_p5_1x1"), feats):
        conv = getattr(m.fpn, name)
        if isinstance(conv, torch.nn.Sequential):     # group_norm: GN normalises the lateral's scale itself
            continue
        rms = F.conv2d(f, cpu(conv.weight)).pow(2).mean().sqrt().item()
        conv.weight.mul_(1.0 / max(rms, 1e-6))


def synthetic_input(H=1024, W=2048, seed=0, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    data = (torch.randn(1, 3, H, W, generator=g) * 50).to(device)   # mean-subtracted BGR scale
    return {"data": data, "im_info": np.array([[H, W, 1.0]], np.float32)}
