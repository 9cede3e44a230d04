"""-m gpu: bf16 wgmma NatureCNN path vs a torch fp32 reference of the same network
(floating-point kernel => torch fp32 reference; tolerance = bf16 operand rounding, stated per check).

Layer-by-layer: the activation workspace is read back and compared against torch's NCHW activations
permuted to NHWC, then every parameter gradient against autograd."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a = a.detach().float().cpu().double(); b = b.detach().float().cpu().double()
    return ((a - b).norm() / max(b.norm().item(), 1e-30)).item()


def _maxrel(a, b):
    a = a.detach().float().cpu().double(); b = b.detach().float().cpu().double()
    return ((a - b).abs().max() / max(b.abs().max().item(), 1e-30)).item()


class _Envs:
    def __init__(self, A):
        from cleanrl_b200.synthetic_envs import Box, Discrete
        self.single_observation_space = Box(0, 255, (4, 84, 84), np.uint8)
        self.single_action_space = Discrete(A)


def _bf16_round(t):
    return t.to(torch.bfloat16).float()


def _limb_round(w):
    """conv1 weights as the integer tensor-core path represents them: per output channel two signed 8-bit limbs,
    w ~= s (l1 / 2^7 + l2 / 2^14) with s = max|w| * 128 / 127 (csrc/tc_conv1_u8.cuh::tc_pack_conv1_i8)."""
    mx = w.abs().flatten(1).max(1).values.view(-1, 1, 1, 1)
    s = torch.where(mx > 0, mx * (128.0 / 127.0), torch.ones_like(mx))
    u = w / s * 128.0
    l1 = torch.clamp(torch.round(u), -127, 127)
    l2 = torch.clamp(torch.round((u - l1) * 128.0), -127, 127)
    return s * (l1 / 128.0 + l2 / 16384.0)


@pytest.mark.parametrize("n,B,A", [(24, 64, 4), (130, 130, 6), (1, 3, 4), (300, 300, 18), (70, 70, 9)])
def test_bf16_forward_backward_layerwise(lib, n, B, A):
    from cleanrl_b200.agents import NatureCNNAgent
    torch.manual_seed(1)
    agent = NatureCNNAgent(_Envs(A)).cuda()
    agent.precision = "bf16"
    agent.flat
    sd = {k: v.detach().cpu().clone() for k, v in agent.state_dict().items()}
    g = torch.Generator().manual_seed(2)
    obs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g)
    rows = torch.randperm(B, generator=g)[:n]
    # ---- torch reference with bf16-rounded weights and activations (what the kernels compute), fp32 accumulate
    W = {k: (_bf16_round(v) if k.startswith("network") and k.endswith("weight") else v.clone()).requires_grad_(True)
         for k, v in sd.items()}
    x = obs[rows].float()
    a1 = torch.relu(F.conv2d(x, W["network.0.weight"], None, stride=4) / 255.0 + W["network.0.bias"].view(1, -1, 1, 1))
    a1r = a1 + (_bf16_round(a1) - a1).detach()
    a2 = torch.relu(F.conv2d(a1r, W["network.2.weight"], W["network.2.bias"], stride=2))
    a2r = a2 + (_bf16_round(a2) - a2).detach()
    a3 = torch.relu(F.conv2d(a2r, W["network.4.weight"], W["network.4.bias"], stride=1))
    a3r = a3 + (_bf16_round(a3) - a3).detach()
    hid = torch.relu(F.linear(a3r.flatten(1), W["network.7.weight"], W["network.7.bias"]))
    hidr = hid + (_bf16_round(hid) - hid).detach()
    logits = F.linear(hidr, W["actor.weight"], W["actor.bias"])
    value = F.linear(hidr, W["critic.weight"], W["critic.bias"])
    # ---- kernels
    lg, val = agent.forward_train(obs.cuda(), rows.cuda())
    torch.cuda.synchronize()
    acts = agent._tc.acts(n, 0).view(torch.bfloat16)
    o = n * 28224          # uint8 input: the workspace starts with the space-to-depth frames
    x0 = acts[:o].view(n, 21, 21, 4, 4, 4).float().cpu()          # [n, Y, X, c, sy, sx]
    ref0 = obs[rows].float().view(n, 4, 21, 4, 21, 4).permute(0, 2, 4, 1, 3, 5)
    assert torch.equal(x0, ref0), "space-to-depth frames must be exact"
    got = {}
    for name, shape in (("act1", (n, 10, 10, 128)), ("act2", (n, 9, 9, 64)), ("act3", (n, 7, 7, 64)), ("hid", (n, 512))):
        cnt = int(np.prod(shape))
        got[name] = acts[o:o + cnt].view(shape).float().cpu()
        o += cnt
    # act1 is stored as 2x2 cells: channel = (py*2+px)*32 + c of pixel (2Y+py, 2X+px)
    a1_cells = a1.view(n, 32, 10, 2, 10, 2).permute(0, 2, 4, 3, 5, 1).reshape(n, 10, 10, 128)
    errs = {
        "act1": _maxrel(got["act1"], a1_cells),
        "act2": _maxrel(got["act2"], a2.permute(0, 2, 3, 1)),
        "act3": _maxrel(got["act3"], a3.permute(0, 2, 3, 1)),
        "hid": _maxrel(got["hid"], hid),
        "logits": _maxrel(lg, logits),
        "value": _maxrel(val, value[:, 0]),
    }
    print("forward max-rel errors:", errs)
    # bf16 output rounding = 2^-9 relative per element; accumulated differences stay below 1e-2 of the tensor max
    for k, v in errs.items():
        assert v < 1e-2, (k, errs)
    # ---- backward
    gl = torch.randn(n, A, generator=g)
    gv = torch.randn(n, generator=g)
    dhead, dl, dv = agent.alloc_head_grad(n, torch.device("cuda"))
    dl.copy_(gl); dv.copy_(gv)
    agent.backward(dhead)
    torch.cuda.synchronize()
    ((logits * gl).sum() + (value[:, 0] * gv).sum()).backward()
    gerrs = {}
    for k, p in agent.named_parameters():
        gerrs[k] = _rel(p.grad, W[k].grad)
    print("gradient rel-L2 errors:", gerrs)
    # activation gradients are rounded to bf16 between layers (2^-9 each): 2e-2 relative L2 per tensor
    for k, v in gerrs.items():
        assert v < 2e-2, (k, gerrs)
    # padded-grid gradient buffers: positions no kernel writes must still be zero
    o = n * (28224 + 12800 + 5184 + 3136 + 512 + 512)
    d3a = acts[o:o + n * 5184].view(n, 9, 9, 64).float().cpu(); o += n * 5184
    d3b = acts[o:o + n * 7744].view(n, 11, 11, 64).float().cpu(); o += n * 7744
    d2a = acts[o:o + n * 6400].view(n, 10, 10, 64).float().cpu(); o += n * 6400
    d2b = acts[o:o + n * 7744].view(n, 11, 11, 64).float().cpu(); o += n * 7744
    d1 = acts[o:o + n * 14112].view(n, 21, 21, 32).float().cpu()
    assert torch.equal(d3a[:, :7, :7], d3b[:, 2:9, 2:9]) and d3a[:, 7:].abs().sum() == 0 and d3a[:, :, 7:].abs().sum() == 0
    assert torch.equal(d2a[:, :9, :9], d2b[:, 1:10, 1:10]) and d2a[:, 9].abs().sum() == 0 and d2a[:, :, 9].abs().sum() == 0
    assert d2b[:, 0].abs().sum() == 0 and d2b[:, 10].abs().sum() == 0 and d2b[:, :, 0].abs().sum() == 0
    assert d1[:, 20].abs().sum() == 0 and d1[:, :, 20].abs().sum() == 0 and torch.isfinite(d1).all()
    assert d1.abs().sum() > 0 and d2a.abs().sum() > 0 and d3a.abs().sum() > 0


def test_s2d_input_equals_uint8_input(lib):
    """Pre-converted space-to-depth frames (engine path) and raw uint8 frames (drop-in path) give identical
    outputs and gradients, with and without the minibatch row gather."""
    from cleanrl_b200 import ops
    from cleanrl_b200.agents import NatureCNNAgent
    torch.manual_seed(2)
    agent = NatureCNNAgent(_Envs(4)).cuda()
    agent.precision = "bf16"
    B, n = 96, 40
    obs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8).cuda()
    rows = torch.randperm(B)[:n].cuda()
    s2d = ops.frames_to_s2d(obs)
    outs, grads = [], []
    for x in (obs, s2d):
        lg, v = agent.forward_train(x, rows)
        dhead, dl, dv = agent.alloc_head_grad(n, torch.device("cuda"))
        dl.copy_(torch.ones(n, 4, device="cuda") * 0.1); dv.copy_(torch.linspace(-1, 1, n, device="cuda"))
        agent.backward(dhead)
        outs.append((lg.clone(), v.clone())); grads.append(agent.flat.grad.clone())
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert torch.equal(grads[0], grads[1])


def test_bf16_rollout_path_matches_fp32_path(lib):
    """Same agent, same frames: the tensor-core path and the exact fp32 path agree to bf16 accuracy,
    and with identical noise they sample the same actions except where p/q is within bf16 error."""
    from cleanrl_b200.agents import NatureCNNAgent
    torch.manual_seed(5)
    agent = NatureCNNAgent(_Envs(4)).cuda()
    obs = torch.randint(0, 256, (1024, 4, 84, 84), dtype=torch.uint8).cuda()
    q = torch.empty(1024, 4, device="cuda").exponential_(1)
    agent.noise_fn = lambda n, A, d: q
    agent.precision = "fp32"
    a32, lp32, _, v32 = agent.get_action_and_value(obs)
    agent.precision = "bf16"
    a16, lp16, _, v16 = agent.get_action_and_value(obs)
    assert (v32 - v16).abs().max().item() < 2e-2 * max(1.0, v32.abs().max().item())
    assert (lp32 - lp16).abs().max().item() < 2e-2
    assert (a32 != a16).float().mean().item() < 0.02


def test_full_size_minibatch_properties(lib):
    """Size-independent properties at BASELINE.json's full minibatch (M = 32 768 rows gathered from a 131 072-frame
    rollout, sorted indices as the engine passes them):
      * batch invariance: a row's logits/value do not depend on which other rows share its tiles -- the first and
        last 64 rows of the big batch equal a 64-row batch of the same frames bit for bit;
      * additivity: the gradient of the full minibatch equals the sum of the gradients of its four quarters
        (different tile/CTA partition and split reduction order => fp32 re-association only)."""
    from cleanrl_b200 import ops
    from cleanrl_b200.agents import NatureCNNAgent
    torch.manual_seed(7)
    dev = torch.device("cuda")
    agent = NatureCNNAgent(_Envs(4)).to(dev)
    agent.precision = "bf16"
    B, M = 131072, 32768
    pool = torch.randint(0, 256, (256, 4, 84, 84), dtype=torch.uint8, device=dev)
    s2d_pool = ops.frames_to_s2d(pool)
    roll = s2d_pool[torch.randint(0, 256, (B,), device=dev)].contiguous()          # [B,21,21,64] bf16, 7.4 GB
    inds = torch.randperm(B, device=dev)[:M].sort().values.contiguous()
    lg, v = agent.forward_train(roll, inds)
    lg, v = lg.clone(), v.clone()
    g = torch.Generator(device="cpu").manual_seed(1)
    dl_all = (torch.randn(M, 4, generator=g) * 1e-3).to(dev); dv_all = (torch.randn(M, generator=g) * 1e-3).to(dev)
    dhead, dl, dv = agent.alloc_head_grad(M, dev)
    dl.copy_(dl_all); dv.copy_(dv_all)
    agent.backward(dhead)
    g_full = agent.flat.grad.clone()
    for sl in (slice(0, 64), slice(M - 64, M)):
        lg_s, v_s = agent.forward_train(roll, inds[sl].contiguous())
        assert torch.equal(lg_s, lg[sl]) and torch.equal(v_s, v[sl])
    g_sum = torch.zeros_like(g_full)
    Q = M // 4
    for q in range(4):
        sl = slice(q * Q, (q + 1) * Q)
        agent.forward_train(roll, inds[sl].contiguous())
        dh, dlq, dvq = agent.alloc_head_grad(Q, dev)
        dlq.copy_(dl_all[sl]); dvq.copy_(dv_all[sl])
        agent.backward(dh)
        g_sum += agent.flat.grad
    rel = ((g_sum - g_full).double().norm() / g_full.double().norm()).item()
    assert rel < 1e-4, rel
    assert torch.isfinite(g_full).all() and g_full.abs().max().item() > 0


@pytest.mark.parametrize("gscale", [1.0, 1e-3])
@pytest.mark.parametrize("n,B,A", [(24, 64, 4), (130, 130, 6), (1, 3, 4), (300, 300, 18), (37, 1000, 4)])
def test_u8_rollout_forward_backward_layerwise(lib, n, B, A, gscale):
    """The uint8 rollout format (what the engine stores and bench.py times): frames as 1-byte space-to-depth pixels in two
    orientations, conv1 forward on the integer tensor cores (exact pixels, two signed 8-bit weight limbs, exact s32
    accumulation), conv1 weight gradient with the pixels converted uint8 -> fp16 in registers and fed from tensor memory.
    Reference = torch fp32 evaluated with the operands the kernels use: bf16-rounded conv2/conv3/fc weights and inter-layer
    activations, conv1 weights as their two-limb representation (5.6e-5 relative L2 from the fp32 master weights, 30x
    closer than bf16).  Emulating the operand rounding matters for the GRADIENT comparison: a ReLU whose pre-activation
    sits within the rounding error of zero flips its mask, and a fraction f of flipped units moves the gradient by
    ~sqrt(f) in relative L2 (2-5 % for f ~ 1e-3), which would mask real kernel errors."""
    from cleanrl_b200 import ops
    from cleanrl_b200.agents import NatureCNNAgent
    torch.manual_seed(1)
    agent = NatureCNNAgent(_Envs(A)).cuda()
    agent.precision = "bf16"
    agent.flat
    sd = {k: v.detach().cpu().clone() for k, v in agent.state_dict().items()}
    g = torch.Generator().manual_seed(2)
    obs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g)
    rows = torch.randperm(B, generator=g)[:n].sort().values
    rm, cm = ops.frames_to_s2d_u8(obs.cuda())
    # layouts: rm[i, Y*21+X, c*16+sy*4+sx] = obs[i, c, 4Y+sy, 4X+sx]; cm[i, ch, pos] likewise, rows 441..447 zero
    ref_rm = obs.view(B, 4, 21, 4, 21, 4).permute(0, 2, 4, 1, 3, 5).reshape(B, 441, 64)
    assert torch.equal(rm.cpu(), ref_rm), "row-major uint8 space-to-depth frames must be exact"
    assert torch.equal(cm.cpu()[:, :, :441], ref_rm.permute(0, 2, 1)) and cm.cpu()[:, :, 441:].abs().sum() == 0
    W = {k: (_limb_round(v) if k == "network.0.weight" else
             _bf16_round(v) if k.startswith("network") and k.endswith("weight") else v.clone()).requires_grad_(True)
         for k, v in sd.items()}
    x = obs[rows].float()
    a1 = torch.relu(F.conv2d(x, W["network.0.weight"], None, stride=4) / 255.0 + W["network.0.bias"].view(1, -1, 1, 1))
    a1r = a1 + (_bf16_round(a1) - a1).detach()
    a2 = torch.relu(F.conv2d(a1r, W["network.2.weight"], W["network.2.bias"], stride=2))
    a2r = a2 + (_bf16_round(a2) - a2).detach()
    a3 = torch.relu(F.conv2d(a2r, W["network.4.weight"], W["network.4.bias"], stride=1))
    a3r = a3 + (_bf16_round(a3) - a3).detach()
    hid = torch.relu(F.linear(a3r.flatten(1), W["network.7.weight"], W["network.7.bias"]))
    hidr = hid + (_bf16_round(hid) - hid).detach()
    logits = F.linear(hidr, W["actor.weight"], W["actor.bias"])
    value = F.linear(hidr, W["critic.weight"], W["critic.bias"])
    lg, val = agent.forward_train(rm, rows.cuda(), aux=cm)
    torch.cuda.synchronize()
    acts = agent._tc.acts(n, 2).view(torch.bfloat16)
    o = 0
    got = {}
    for name, shape in (("act1", (n, 10, 10, 128)), ("act2", (n, 9, 9, 64)), ("act3", (n, 7, 7, 64)), ("hid", (n, 512))):
        cnt = int(np.prod(shape))
        got[name] = acts[o:o + cnt].view(shape).float().cpu()
        o += cnt
    a1_cells = a1.view(n, 32, 10, 2, 10, 2).permute(0, 2, 4, 3, 5, 1).reshape(n, 10, 10, 128)
    errs = {"act1": _maxrel(got["act1"], a1_cells), "act2": _maxrel(got["act2"], a2.permute(0, 2, 3, 1)),
            "act3": _maxrel(got["act3"], a3.permute(0, 2, 3, 1)), "hid": _maxrel(got["hid"], hid),
            "logits": _maxrel(lg, logits), "value": _maxrel(val, value[:, 0])}
    print("u8 rollout forward max-rel errors:", errs)
    assert errs["act1"] < 4e-3, errs          # bf16 OUTPUT rounding only (2^-9): inputs exact, weights to 2^-15 of the row max
    for k, v in errs.items():
        assert v < 1e-2, (k, errs)
    gl = torch.randn(n, A, generator=g) * gscale        # 1e-3: realistic magnitudes (the loss is a mean over 32 768 samples)
    gv = torch.randn(n, generator=g) * gscale
    dhead, dl, dv = agent.alloc_head_grad(n, torch.device("cuda"))
    dl.copy_(gl); dv.copy_(gv)
    agent.backward(dhead)
    torch.cuda.synchronize()
    ((logits * gl).sum() + (value[:, 0] * gv).sum()).backward()
    gerrs = {k: _rel(p.grad, W[k].grad) for k, p in agent.named_parameters()}
    print("u8 rollout gradient rel-L2 errors:", gerrs)
    for k, v in gerrs.items():
        assert v < 2e-2, (k, gerrs)
    assert torch.isfinite(agent.flat.grad).all()


def test_u8_rollout_equals_bf16_rollout_downstream(lib):
    """Both rollout layouts hold the same pixels exactly; their conv1 outputs differ only by the weight representation
    (two 8-bit limbs vs one bf16), so heads and gradients agree to bf16 accuracy, with and without the row gather."""
    from cleanrl_b200 import ops
    from cleanrl_b200.agents import NatureCNNAgent
    torch.manual_seed(2)
    agent = NatureCNNAgent(_Envs(4)).cuda()
    agent.precision = "bf16"
    B, n = 96, 40
    obs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8).cuda()
    s2d = ops.frames_to_s2d(obs)
    rm, cm = ops.frames_to_s2d_u8(obs)
    for rows in (torch.randperm(B)[:n].sort().values.cuda(), None):
        m = n if rows is not None else B
        res = []
        for x, aux in ((s2d, None), (rm, cm)):
            lg, v = agent.forward_train(x, rows, **({"aux": aux} if aux is not None else {}))
            dhead, dl, dv = agent.alloc_head_grad(m, torch.device("cuda"))
            dl.copy_(torch.ones(m, 4, device="cuda") * 1e-3); dv.copy_(torch.linspace(-1, 1, m, device="cuda") * 1e-3)
            agent.backward(dhead)
            res.append((lg.clone(), v.clone(), agent.flat.grad.clone()))
        assert _maxrel(res[1][0], res[0][0]) < 1e-2 and _maxrel(res[1][1], res[0][1]) < 1e-2
        assert _rel(res[1][2], res[0][2]) < 2e-2
