"""The tensor-core IMPALA-CNN (csrc/net_impala_tc.cu) against an fp64 emulator of the same network, layer by layer.

Integer-exact mode: every weight is 0 or +-1, every bias -1, 0 or 1 (the seq0 conv's 0), every pixel 0 or 255 and the
head gradient 0 or +-1 on a few hundred "live" rows.  Every fp32 reduction of the kernels then adds integers whose absolute
values sum to less than 2^24 (the emulator returns those sums and the test asserts the bound), so every partial sum is
exact in any order: the mma.sync accumulations, the weight gradients' per-CTA partials and their fold.  The kernels must
then equal the emulator bit for bit (bf16 rounded at the same points, RNE) in every stored tensor, the head outputs and
every parameter gradient, at every batch size: a dropped, duplicated or misplaced term fails at any n, in any band
group or CTA range.

Realistic mode: torch's default initialisation and uniform pixels.  Each layer is recomputed in fp64 from the tensors
the kernels stored for its inputs and compared within half a bf16 ulp plus 1e-4 of its sum of |products|, which
catches rounding-mode errors that integers cannot show.

The CPU tests check the emulator itself against torch autograd and the integer generator against the 2^24 budget."""
import math

import pytest
import torch
import torch.nn.functional as F

from test_gpu_procgen import _Envs, _ref_forward

A = 15
BUDGET = 2.0 ** 24
SCALE = float(torch.tensor(1.0 / 255.0, dtype=torch.float32))     # the fp32 1/255 of the seq0 conv and its gradient
WGRAD_CTAS = 264                                                 # kWgradCtas: row splits of the conv weight gradients
CHUNK = 256                                                      # images per emulator pass
# band geometry of each conv stage: (bands per image, bands per group) -- geo() in net_impala_tc.cu
STAGES = {"64x64 (seq0)": (16, 1), "32x32": (4, 1), "16x16": (1, 1), "8x8": (1, 3)}
INT_SIZES = [1, 2, 5, 16, 17, 66, 67, 264, 265, 792, 793, 512, 1024, 2048, 8192, 16384]


# ---------------------------------------------------------------- fp64 emulator (channel-last tensors [B, H, W, C])
def _bf(t):
    """An fp32 result stored as bf16 (round to nearest even)."""
    return t.to(torch.float32).to(torch.bfloat16).to(torch.float64)


def _f32(t):
    return t.to(torch.float32).to(torch.float64)


def _ident(t):
    return t


def _conv(x, w):
    """3x3, pad-1 convolution of x [B, H, W, Ci] with a torch-layout weight [Co, Ci, 3, 3]: nine shifted GEMMs."""
    _, H, W, _ = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    out = 0
    for ky in range(3):
        for kx in range(3):
            out = out + xp[:, ky:ky + H, kx:kx + W, :] @ w[:, :, ky, kx].t()
    return out


def _flip_t(w):
    """The data gradient's weight: a 3x3 convolution of dY with w[co, ci, 2 - ky, 2 - kx] as [ci, co, ky, kx]."""
    return w.flip(2, 3).transpose(0, 1)


def _wgrad(x, dy):
    """(dW [Co, Ci, 3, 3], db [Co]) of a 3x3, pad-1 convolution with input x and output gradient dy."""
    _, H, W, Ci = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    d = dy.reshape(-1, dy.shape[-1]).t()
    gw = x.new_empty(dy.shape[-1], Ci, 3, 3)
    for ky in range(3):
        for kx in range(3):
            gw[:, :, ky, kx] = d @ xp[:, ky:ky + H, kx:kx + W, :].reshape(-1, Ci)
    return gw, dy.sum((0, 1, 2))


def _pool_windows(x):
    """[B, OH, OW, C, 9]: the 3x3 / stride-2 / pad-1 windows in row-major tap order, -inf outside the image."""
    _, H, W, _ = x.shape
    OH, OW = (H + 1) // 2, (W + 1) // 2
    xp = F.pad(x, (0, 0, 1, 1, 1, 1), value=-math.inf)
    return torch.stack([xp[:, ky:ky + 2 * OH:2, kx:kx + 2 * OW:2, :] for ky in range(3) for kx in range(3)], -1)


def _maxpool(x):
    """(max, tap of the FIRST maximum in row-major window order)."""
    win = _pool_windows(x)
    arg = win.argmax(-1)
    return win.gather(-1, arg[..., None])[..., 0], arg


def _maxpool_bwd(dy, arg, H, W):
    B, OH, OW, C = dy.shape
    dxp = dy.new_zeros(B, H + 2, W + 2, C)
    for k in range(9):
        ky, kx = divmod(k, 3)
        dxp[:, ky:ky + 2 * OH:2, kx:kx + 2 * OW:2, :] += dy * (arg == k)
    return dxp[:, 1:H + 1, 1:W + 1, :]


def _bits(t):
    """int32 words [B, K / 32]: bit k of word j = t[:, 32 j + k] > 0 (the kernels' ReLU mask words)."""
    B, K = t.shape
    w = ((t > 0).view(B, K // 32, 32).long() << torch.arange(32, device=t.device)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def _fc_packed(w):
    """fc weight [256, c*64 + p] (torch's NCHW flatten) -> [256, p*32 + c] (the channel-last stream's K order)."""
    return w.view(256, 32, 64).transpose(1, 2).reshape(256, 2048)


def _fc_unpacked(w):
    return w.view(256, 64, 32).transpose(1, 2).reshape(256, 2048)


def emulate(P, obs, dhead=None, rnd=True, stored=None, skip_col=None, round_out=True):
    """ImpalaAgent / PPGAgent on frames ``obs`` [B, 64, 64, 3] in fp64, laid out and rounded as the kernels do.

    ``P``: fp64 parameters by state_dict name, with the joint head as ``head.weight`` [A1, 256] / ``head.bias``.
    ``rnd``: round conv / fc weights and the stored tensors to bf16 and the fp32 results to fp32 where the kernels do
    (False: exact fp64 of the same network); ``round_out`` = False keeps each layer's own output exact (the reference
    the realistic mode compares with) while the weights stay rounded.  ``stored``: tensors (emulator names and shapes)
    that replace the emulator's own as the inputs of the layers that read them, so that each layer is checked on the
    kernels' inputs.
    ``skip_col``: head column left out of the hidden layer's gradient (PPG's critic).

    Returns (T, Ta, out, grads, grads_abs, budget): the stored tensors by ``act_tensors`` name (the backward buffers
    ga / gb / gy / dc as they are at the end of the backward: d(s0_0), d(s1_0), d(y0_0), d(c0)), their sums of
    |products|, the head output [B, A1], the parameter gradients by state_dict name and their sums of |products| (the
    seq0 conv weight's as summed, before fold_seq0's 1/255), and the largest sum of |products| of any per-image
    reduction."""
    R, R32 = (_bf, _f32) if rnd and round_out else (_ident, _ident)
    Wr = _bf if rnd else _ident
    scale = SCALE if rnd else 1.0 / 255.0
    S = (lambda name, own: stored[name].reshape(own.shape) if stored is not None and name in stored else own)
    T, Ta, G, Ga, red = {}, {}, {}, {}, []
    B = obs.shape[0]
    x = obs.to(torch.float64)
    xin, blocks = [], {}
    # ---- forward
    for q in range(3):
        pre = f"network.{q}"
        w, b = Wr(P[f"{pre}.conv.weight"]), P[f"{pre}.conv.bias"]
        if q:
            x = S(f"s2_{q - 1}", x)
        xin.append(x)
        acc, acca = _conv(x, w), _conv(x.abs(), w.abs())
        red.append(acca.max())
        if q == 0:
            T["c0"], Ta["c0"] = R(R32(acc * scale + b)), acca * scale + b.abs()        # fmaf(acc, 1/255, b)
        else:
            T[f"c{q}"], Ta[f"c{q}"] = R(R32(acc + b)), acca + b.abs()
        c = S(f"c{q}", T[f"c{q}"])
        s, arg = _maxpool(c)
        T[f"s0_{q}"], T[f"arg_{q}"] = s, arg
        for blk in (0, 1):
            rb = f"{pre}.res_block{blk}"
            s = S(f"s{blk}_{q}", s)
            rs = s.clamp(min=0)                                        # conv0 stages relu(x)
            w0, b0 = Wr(P[f"{rb}.conv0.weight"]), P[f"{rb}.conv0.bias"]
            acc, acca = _conv(rs, w0), _conv(rs, w0.abs())
            red.append(acca.max())
            T[f"y{blk}_{q}"], Ta[f"y{blk}_{q}"] = R(R32(acc + b0).clamp(min=0)), acca + b0.abs()
            y = S(f"y{blk}_{q}", T[f"y{blk}_{q}"])
            blocks[(q, blk)] = (s, y)
            w1, b1 = Wr(P[f"{rb}.conv1.weight"]), P[f"{rb}.conv1.bias"]
            acc, acca = _conv(y, w1), _conv(y, w1.abs())
            t, ta = R32(R32(acc + b1) + s), acca + b1.abs() + s.abs()  # bf16(x + acc + b), summed in fp32
            red.append(ta.max())
            if q == 2 and blk == 1:                                    # relu(stream) = the fc input, packed K order
                T["h0"], Ta["h0"] = R(t.clamp(min=0)).reshape(B, 2048), ta.reshape(B, 2048)
                T["mh0"] = _bits(T["h0"])
            else:
                s = R(t)
                T[f"s{blk + 1}_{q}"], Ta[f"s{blk + 1}_{q}"] = s, ta
        x = s
    h0 = S("h0", T["h0"])
    wfc, bfc = _fc_packed(Wr(P["network.5.weight"])), P["network.5.bias"]
    acca = h0 @ wfc.abs().t() + bfc.abs()
    red.append(acca.max())
    T["hid"], Ta["hid"] = R(R32(h0 @ wfc.t() + bfc).clamp(min=0)), acca
    T["mhid"] = _bits(T["hid"])
    hid = S("hid", T["hid"])
    wh, bh = P["head.weight"], P["head.bias"]
    out, outa = R32(hid @ wh.t() + bh), hid @ wh.abs().t() + bh.abs()
    red.append(outa.max())
    if dhead is None:
        return T, Ta, (out, outa), G, Ga, max(r.item() for r in red)
    # ---- backward
    dh = dhead.to(torch.float64)
    G["head.weight"], Ga["head.weight"] = dh.t() @ hid, dh.abs().t() @ hid
    G["head.bias"], Ga["head.bias"] = dh.sum(0), dh.abs().sum(0)
    dhh = dh.clone()
    if skip_col is not None:
        dhh[:, skip_col] = 0                                           # critic(hidden.detach())
    acca = dhh.abs() @ wh.abs()
    red.append(acca.max())
    T["dhid"], Ta["dhid"] = R(R32(dhh @ wh) * (hid > 0)), acca
    dhid = S("dhid", T["dhid"])
    G["network.5.weight"], Ga["network.5.weight"] = _fc_unpacked(dhid.t() @ h0), _fc_unpacked(dhid.abs().t() @ h0)
    G["network.5.bias"], Ga["network.5.bias"] = dhid.sum(0), dhid.abs().sum(0)
    ga = dhid.abs() @ wfc.abs()
    red.append(ga.max())
    g = R(R32(dhid @ wfc) * (h0 > 0)).view(B, 8, 8, 32)              # d(stream) of the last block
    for q in (2, 1, 0):
        pre = f"network.{q}"
        for blk in (1, 0):
            rb = f"{pre}.res_block{blk}"
            if q == 0 and blk == 0:
                T["gb"] = g
                g = S("gb", g)
            s, y = blocks[(q, blk)]
            w0, w1 = Wr(P[f"{rb}.conv0.weight"]), Wr(P[f"{rb}.conv1.weight"])
            G[f"{rb}.conv1.weight"], G[f"{rb}.conv1.bias"] = _wgrad(y, g)
            Ga[f"{rb}.conv1.weight"], Ga[f"{rb}.conv1.bias"] = _wgrad(y, g.abs())
            gya = _conv(g.abs(), _flip_t(w1).abs())
            red.append(gya.max())
            gy = R(R32(_conv(g, _flip_t(w1))) * (y > 0))
            if q == 0 and blk == 0:
                T["gy"], Ta["gy"] = gy, gya
                gy = S("gy", gy)
            rs = s.clamp(min=0)
            G[f"{rb}.conv0.weight"], G[f"{rb}.conv0.bias"] = _wgrad(rs, gy)
            Ga[f"{rb}.conv0.weight"], Ga[f"{rb}.conv0.bias"] = _wgrad(rs, gy.abs())
            gna = _conv(gy.abs(), _flip_t(w0).abs()) + g.abs()
            red.append(gna.max())
            g = R(R32(R32(_conv(gy, _flip_t(w0))) * (s > 0) + g))    # mask, then the skip gradient
        if q == 0:
            T["ga"], Ta["ga"] = g, gna
            g = S("ga", g)
        H = 64 >> q
        arg = S(f"arg_{q}", T[f"arg_{q}"])
        dc, dca = R(R32(_maxpool_bwd(g, arg, H, H))), _maxpool_bwd(g.abs(), arg, H, H)
        if q == 0:
            T["dc"], Ta["dc"] = dc, dca
            dc = S("dc", dc)
        wc = Wr(P[f"{pre}.conv.weight"])
        gw, gb = _wgrad(xin[q], dc)
        Ga[f"{pre}.conv.weight"], Ga[f"{pre}.conv.bias"] = _wgrad(xin[q].abs(), dc.abs())
        G[f"{pre}.conv.weight"], G[f"{pre}.conv.bias"] = gw, gb
        if q:
            red.append(_conv(dc.abs(), _flip_t(wc).abs()).max())
            g = R(R32(_conv(dc, _flip_t(wc))))
    for k in ("ga", "gb", "gy", "dc"):
        T[k] = T[k].reshape(B, -1)
        if k in Ta:
            Ta[k] = Ta[k].reshape(B, -1)
    return T, Ta, (out, outa), G, Ga, max(r.item() for r in red)


def fold_seq0(G, rnd=True):
    """The seq0 conv weight gradient of the summed pixel products: fold_conv's one fp32 rounding of sum * fp32(1/255)."""
    k = "network.0.conv.weight"
    return {**G, k: _f32(G[k] * SCALE) if rnd else G[k] / 255.0}


def params_of(agent):
    """fp64 parameters by state_dict name, the joint head as ``head.weight`` / ``head.bias``."""
    sd = {k: v.detach().to(torch.float64) for k, v in agent.state_dict().items()}
    heads = [h for h in ("actor", "critic", "aux_critic") if f"{h}.weight" in sd]
    P = {k: v for k, v in sd.items() if not k.split(".")[0] in heads}
    P["head.weight"] = torch.cat([sd[f"{h}.weight"] for h in heads])
    P["head.bias"] = torch.cat([sd[f"{h}.bias"] for h in heads])
    return P, heads


def split_head_grads(G, heads):
    out = {k: v for k, v in G.items() if not k.startswith("head.")}
    for kind in ("weight", "bias"):
        rows = G[f"head.{kind}"]
        out[f"actor.{kind}"] = rows[:A]
        for j, h in enumerate(heads[1:]):
            out[f"{h}.{kind}"] = rows[A + j:A + j + 1]
    return out


# ---------------------------------------------------------------- integer operands
def int_params(named, gen):
    """+-1 weights at about 1.5 nonzero terms per output, biases in {-1, 0, 1}; the seq0 conv bias 0, so that
    fmaf(255 k, fp32(1/255), 0) rounds back to k once stored as bf16."""
    out = {}
    for name, shape in named:
        if name.endswith("weight"):
            p = (1.5 / (9 * shape[1]) if len(shape) == 4 else 6.0 / 2048 if shape[1] == 2048 else 8.0 / 256)
        else:
            p = 0.0 if name == "network.0.conv.bias" else 0.25
        sign = torch.randint(0, 2, shape, generator=gen).to(torch.float32) * 2 - 1
        out[name] = sign * (torch.rand(shape, generator=gen) < p)
    return out


def int_frames(B, gen, device=None):
    """uint8 frames [B, 64, 64, 3]: 3 % of the pixels 255, the rest 0."""
    return ((torch.rand(B, 64, 64, 3, generator=gen, device=device) < 0.03) * 255).to(torch.uint8)


def live_rows(n):
    """Rows with a nonzero head gradient: every ceil(n / 264)-th row and the last one."""
    step = -(-n // WGRAD_CTAS)
    rows = list(range(0, n, step))
    return rows + [n - 1] if rows[-1] != n - 1 else rows


def int_dhead(n, A1, gen, device=None, live=None):
    """Head gradient [n, A1]: +-1 at half the entries of the live rows (default live_rows(n)), 0 elsewhere."""
    d = torch.zeros(n, A1)
    live = live_rows(n) if live is None else live
    sign = torch.randint(0, 2, (len(live), A1), generator=gen).to(torch.float32) * 2 - 1
    d[live] = sign * (torch.rand(len(live), A1, generator=gen) < 0.5)
    return d.to(device) if device is not None else d


def wgrad_cta_images(n, bpi, nb):
    """[(first image, last image)] touched by each weight-gradient CTA's band-group range (run_wgrad's split)."""
    nbands = n * bpi
    groups = -(-nbands // nb)
    ctas = min(groups, WGRAD_CTAS)
    per = -(-groups // ctas)
    out = []
    for g0 in range(0, groups, per):
        b0, b1 = g0 * nb, min((g0 + per) * nb, nbands)
        out.append((b0 // bpi, (b1 - 1) // bpi))
    return out


# ---------------------------------------------------------------- CPU tests of the emulator
def _impala(A_=A, seed=2):
    from cleanrl_b200.agents import ImpalaAgent
    torch.manual_seed(seed)
    return ImpalaAgent(_Envs(A_))


def test_emulator_unrounded_equals_fp64_reference_and_autograd():
    n = 3
    agent = _impala()
    g = torch.Generator().manual_seed(3)
    obs = torch.randint(0, 256, (n, 64, 64, 3), dtype=torch.uint8, generator=g)
    dhead = torch.randn(n, A + 1, generator=g, dtype=torch.float64)
    sd = {k: v.detach().double().requires_grad_(True) for k, v in agent.state_dict().items()}
    logits, value = _ref_forward(sd, obs)
    ((logits * dhead[:, :A]).sum() + (value * dhead[:, A]).sum()).backward()
    P, heads = params_of(agent)
    T, _, (out, _), G, _, _ = emulate(P, obs, dhead, rnd=False)
    torch.testing.assert_close(out[:, :A], logits.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(out[:, A], value.detach(), rtol=1e-12, atol=1e-12)
    G = split_head_grads(fold_seq0(G, rnd=False), heads)
    assert set(G) == set(sd)
    for k, v in sd.items():
        torch.testing.assert_close(G[k], v.grad, rtol=1e-10, atol=1e-12 * v.grad.abs().max().item(), msg=k)
    assert set(T) >= {"c0", "c1", "c2", "s1_2", "y1_2", "arg_2", "h0", "mh0", "hid", "mhid", "dhid", "ga", "gb", "gy", "dc"}


def test_emulator_maxpool_takes_first_maximum():
    x = -torch.ones(2, 4, 4, 1, dtype=torch.float64)
    x[0, 0, 1, 0] = x[0, 1, 0, 0] = 2.0                   # window (0, 0): taps 5 and 7 tied at the maximum
    y, arg = _maxpool(x)
    assert arg[0, :, :, 0].tolist() == [[5, 3], [1, 0]]  # the first maximum in row-major tap order
    assert arg[1, 0, 0, 0] == 4                            # -inf padding: the first tap inside the image
    dx = _maxpool_bwd(torch.ones_like(y), arg, 4, 4)
    assert dx[0, 0, 1, 0] == 2 and dx[0, 1, 0, 0] == 1 and dx[0, 1, 1, 0] == 1 and dx[0].sum() == 4


@pytest.mark.parametrize("n", INT_SIZES)
def test_live_rows_reach_every_wgrad_cta(n):
    live = set(live_rows(n))
    for stage, (bpi, nb) in STAGES.items():
        for lo, hi in wgrad_cta_images(n, bpi, nb):
            assert live & set(range(lo, hi + 1)), (stage, lo, hi)


def test_integer_generator_meets_fp32_budget():
    """The largest live-row count of the sizes tested (265), every row live: each reduction's sum of |products| must
    stay below 2^24 (the weight gradients' sums grow with the live rows, the rest are per image)."""
    n = max(len(live_rows(m)) for m in INT_SIZES)
    agent = _impala()
    gen = torch.Generator().manual_seed(11)
    ip = int_params([(k, tuple(v.shape)) for k, v in agent.named_parameters()], gen)
    P = {k: v.double() for k, v in ip.items() if not k.split(".")[0] in ("actor", "critic")}
    P["head.weight"] = torch.cat([ip["actor.weight"], ip["critic.weight"]]).double()
    P["head.bias"] = torch.cat([ip["actor.bias"], ip["critic.bias"]]).double()
    obs = int_frames(n, gen)
    dhead = int_dhead(n, A + 1, gen, live=list(range(n)))
    Ga, worst, hid_pos = None, 0.0, []
    for i0 in range(0, n, 64):
        T, _, _, _, ga, red = emulate(P, obs[i0:i0 + 64], dhead[i0:i0 + 64])
        Ga = ga if Ga is None else {k: Ga[k] + v for k, v in ga.items()}
        worst = max(worst, red)
        hid_pos.append((T["hid"] > 0).double().mean().item())
    worst = max(worst, max(v.max().item() for v in Ga.values()))
    assert worst < BUDGET, worst
    assert 0.2 < sum(hid_pos) / len(hid_pos) < 0.8          # the ReLU masks stay mixed


# ---------------------------------------------------------------- GPU: the kernels against the emulator
def _diff_report(name, got, ref, i0, rows):
    """Where ``got`` and ``ref`` (batch rows i0 + ...) differ: count, batch rows and their 8x8 band groups, first values."""
    bad = (got != ref).nonzero()
    idx = bad[:5].tolist()
    where = [f"{tuple(i)}: {got[tuple(i)].item()} != {ref[tuple(i)].item()}" for i in idx]
    if rows is False:                                      # a parameter gradient: no batch rows
        return f"{name}: {bad.shape[0]} of {ref.numel()} differ; first at {where}"
    imgs = sorted({i0 + int(r) for r in bad[:, 0].tolist()})
    return (f"{name}: {bad.shape[0]} of {ref.numel()} differ; batch rows {imgs[:12]}{'...' if len(imgs) > 12 else ''} "
            f"(8x8 band groups {sorted({r // 3 for r in imgs})[:12]}); first at (row - {i0}, ...) {where}"
            + (f"; frame indices {[int(rows[r]) for r in imgs[:6]]}" if rows is not None else ""))


def _kernel_chunk(K, sl, T):
    """The kernels' stored tensors of batch rows ``sl``, shaped and typed like the emulator's."""
    out = {}
    for name, ref in T.items():
        got = K[name][sl].reshape(ref.shape)
        out[name] = got.long() if name.startswith("arg_") else got if got.dtype == torch.int32 else got.double()
    return out


def _run_agent(agent, obs, rows, dhead, aux):
    """Forward + backward on the agent's bf16 plan; the head output [n, A1] and the gradients by parameter name."""
    if aux:
        out = agent.forward_aux(obs, rows).clone()
    else:
        lg, val = agent.forward_train(obs, rows)
        out = torch.cat([lg, val[:, None]], 1)
    n = out.shape[0]
    dh, _, _ = agent.alloc_head_grad(n, obs.device)
    dh.copy_(dhead)
    agent.backward(dh)
    torch.cuda.synchronize()
    return out, {k: p.grad.detach().clone() for k, p in agent.named_parameters()}


def _make_agent(ppg, seed):
    from cleanrl_b200.agents import ImpalaAgent, PPGAgent
    torch.manual_seed(seed)
    agent = (PPGAgent if ppg else ImpalaAgent)(_Envs(A)).cuda()
    agent.precision = "bf16"
    agent.flat
    return agent


def _integer_exact(n, ppg, gather, seed):
    dev = torch.device("cuda")
    agent = _make_agent(ppg, seed)
    gen = torch.Generator().manual_seed(seed)
    ip = int_params([(k, tuple(p.shape)) for k, p in agent.named_parameters()], gen)
    with torch.no_grad():
        for k, p in agent.named_parameters():
            p.copy_(ip[k])
    agent.params_updated()
    A1 = A + (2 if ppg else 1)
    gdev = torch.Generator(device=dev).manual_seed(seed)
    if gather:
        B = n + n // 3 + 3
        obs = int_frames(B, gdev, dev)
        rows = torch.randperm(B, generator=gdev, device=dev)[:n]
        assert n < 3 or not bool((rows[1:] >= rows[:-1]).all())
    else:
        obs, rows = int_frames(n, gdev, dev), None
    dhead = int_dhead(n, A1, gen, dev)
    out_k, grads_k = _run_agent(agent, obs, rows, dhead, aux=ppg)
    K = agent._tc.act_tensors(n)
    P, heads = params_of(agent)
    G, Ga, worst = None, None, 0.0
    for i0 in range(0, n, CHUNK):
        sl = slice(i0, min(i0 + CHUNK, n))
        frames = obs[rows[sl]] if rows is not None else obs[sl]
        T, _, (out, _), g, ga, red = emulate(P, frames, dhead[sl], skip_col=A if ppg else None)
        worst = max(worst, red)
        Kc = _kernel_chunk(K, sl, T)
        for name, ref in T.items():
            assert torch.equal(Kc[name], ref), _diff_report(name, Kc[name], ref, i0, rows)
        assert torch.equal(out_k[sl].double(), out), _diff_report("head output", out_k[sl].double(), out, i0, rows)
        G = g if G is None else {k: G[k] + v for k, v in g.items()}
        Ga = ga if Ga is None else {k: Ga[k] + v for k, v in ga.items()}
    worst = max(worst, max(v.max().item() for v in Ga.values()))
    assert worst < BUDGET, f"integer operands exceed the exact fp32 range: largest sum of |products| {worst}"
    G = split_head_grads(fold_seq0(G), heads)
    assert set(G) == set(grads_k)
    for k, ref in G.items():
        got = grads_k[k].double().reshape(ref.shape)
        assert torch.equal(got, ref), _diff_report(f"grad {k}", got, ref, 0, False)
    return T


@pytest.mark.gpu
@pytest.mark.parametrize("n,gather", [(n, True) for n in INT_SIZES] + [(265, False)])
def test_impala_integer_exact(lib, n, gather):
    T = _integer_exact(n, ppg=False, gather=gather, seed=n)
    assert (T["hid"] > 0).any() and (T["dhid"] != 0).any()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [5, 1024, 8192])
def test_ppg_integer_exact(lib, n):
    _integer_exact(n, ppg=True, gather=True, seed=n + 1)


def _close(name, got, ref, absum):
    tol = 2.0 ** -8 * ref.abs() + 1e-4 * absum
    bad = (got - ref).abs() > tol
    assert not bad.any(), (f"{name}: {int(bad.sum())} of {ref.numel()} outside half a bf16 ulp + 1e-4 sum|products|; "
                           f"worst excess {((got - ref).abs() - tol).max().item():.3g} at {bad.nonzero()[0].tolist()}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [5, 2048, 16384])
def test_impala_layers_on_stored_inputs(lib, n):
    """Default initialisation, uniform pixels: each layer in fp64 on the kernels' own stored inputs."""
    dev = torch.device("cuda")
    agent = _make_agent(False, seed=7)
    gdev = torch.Generator(device=dev).manual_seed(n)
    B = n + 7
    obs = torch.randint(0, 256, (B, 64, 64, 3), dtype=torch.uint8, generator=gdev, device=dev)
    rows = torch.randperm(B, generator=gdev, device=dev)[:n]
    dhead = torch.randn(n, A + 1, generator=gdev, device=dev)
    out_k, grads_k = _run_agent(agent, obs, rows, dhead, aux=False)
    K = agent._tc.act_tensors(n)
    P, heads = params_of(agent)
    exact = {f"s0_{q}" for q in range(3)} | {f"arg_{q}" for q in range(3)}     # max-pools of the stored conv outputs
    tolerant = {"c0", "c1", "c2", "h0", "hid", "dhid", "gy", "ga", "dc"} | \
        {f"{k}{j}_{q}" for q in range(3) for k, j in (("s", 1), ("s", 2), ("y", 0), ("y", 1)) if (q, k, j) != (2, "s", 2)}
    G, Ga = None, None
    for i0 in range(0, n, CHUNK):
        sl = slice(i0, min(i0 + CHUNK, n))
        names = exact | tolerant | {"gb", "mh0", "mhid"}
        stored = _kernel_chunk(K, sl, {k: _shape_ref(k, sl.stop - sl.start) for k in names})
        T, Ta, (out, outa), g, ga, _ = emulate(P, obs[rows[sl]], dhead[sl], stored=stored, round_out=False)
        for name in exact:
            assert torch.equal(stored[name], T[name]), _diff_report(name, stored[name], T[name], i0, rows)
        for name in tolerant:
            _close(name, stored[name], T[name], Ta[name])
        for bits, t in (("mh0", "h0"), ("mhid", "hid")):                   # the mask words of the stored tensors
            assert torch.equal(stored[bits], _bits(stored[t])), bits
        _close("head output", out_k[sl].double(), out, outa)
        G = g if G is None else {k: G[k] + v for k, v in g.items()}
        Ga = ga if Ga is None else {k: Ga[k] + v for k, v in ga.items()}
    Ga["network.0.conv.weight"] = Ga["network.0.conv.weight"] * SCALE
    G, Ga = split_head_grads(fold_seq0(G), heads), split_head_grads(Ga, heads)
    checked = [f"{h}.{k}" for h in heads for k in ("weight", "bias")] + \
        [f"network.{l}.{k}" for l in ("5", "0.conv", "0.res_block0.conv0", "0.res_block0.conv1") for k in ("weight", "bias")]
    for k in checked:
        _close(f"grad {k}", grads_k[k].double().reshape(G[k].shape), G[k], Ga[k])


def _shape_ref(name, B):
    """A placeholder with the emulator's shape and dtype of tensor ``name`` for B images."""
    shapes = {"c0": (64, 64, 16), "c1": (32, 32, 32), "c2": (16, 16, 32), "h0": (2048,), "mh0": (64,), "hid": (256,),
              "mhid": (8,), "dhid": (256,), "ga": (16384,), "gb": (16384,), "gy": (16384,), "dc": (65536,)}
    if name in shapes:
        dims = shapes[name]
    else:
        q = int(name[-1])
        dims = ((32, 32, 16), (16, 16, 32), (8, 8, 32))[q]
    dtype = torch.int32 if name in ("mh0", "mhid") else torch.int64 if name.startswith("arg_") else torch.float64
    return torch.empty((B,) + dims, dtype=dtype, device="meta")
