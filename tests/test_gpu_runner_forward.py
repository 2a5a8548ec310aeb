"""The ResNet runner's forward pass in place, element by element, against float64: every tensor a training-mode
forward leaves behind, read back through dirb200_resnet_peek, _peek_conv and _peek_bn_stats, teacher-forced (each check
is fed the runner's own stored inputs, taken from where the reference network says they come from, never from a
pointer the runner reports).  u = 2^-24.

  conv output y        float64 conv of the stored bf16 input and the conv's own bf16 fprop operand (the stem: x
                       rounded to bf16 and the 3x7x7 filter read back from the space-to-depth operand, at stride 2,
                       pad 3); every element within 2^-8 |ref| + (1 + 2^-8) KAPPA(K) A, the bound of test_gpu_conv.py.
  mean / invstd        per channel against float64 statistics of the runner's own bf16 y.  The fprop epilogue sums the
                       bf16-ROUNDED outputs (it reads them back from the staging tile, conv_igemm.cu) in an fp32 chain
                       of L = 16 staged rows + the tiles one CTA walks + 3 combine levels, and bn_finalize adds the CTA
                       rows in float64: |S - S_ref| <= L u sum |term|.  With DIRB200_FUSED_STATS=0 the sums come from
                       bn_stats: L = ceil(rows / (CTAs x row lanes)) + lanes + 2.  mean = S0 / n and
                       var = S1 / n - mean^2 carry that error, dm = L u sum|y| / n and
                       dvar = L u sum y^2 / n + 2 |m| dm + dm^2, plus one fp32 rounding of each output; invstd moves by
                       at most dvar / (2 (var + eps)) relative.  The bounds are those of test_gpu_conv_epilogues.py.
  scale / shift        scale = gamma invstd (one fp32 rounding), shift = beta - mean scale (at most two): within
                       u |scale| and u (|shift| + |mean scale|) of float64 arithmetic on the runner's own fp32 mean,
                       invstd and parameters.
  running statistics   every BatchNorm's running_mean / running_var after each forward against float64 from the values
                       before it: momentum 0.1 and the unbiased variance n / (n - 1), within the error the sums carry
                       (momentum x dm, momentum x dvar n / (n - 1)) plus 4 u of each term; num_batches_tracked + 1.
  a1, a2, block output bit-exact: bf16(relu(fl32(y scale + shift) [+ shortcut])), the fmaf formed exactly in float64
                       (the formula of test_gpu_layer_kernels.py's bn_apply references); the shortcut is the block input
                       or fl32(y_ds scale_ds + shift_ds).
  max pool             bit-exact values and the FIRST maximum of each 3x3 window (pool_ref of test_gpu_layer_kernels.py)
                       over bf16(relu(fl32(y scale + shift))) of the stem.
  ReLU masks           every bit equals (block output > 0).  C is a multiple of 8, so a row has no padding bits.
  encoding             the fp32 average pool: |enc - mean| <= ((hw - 1) u sum|x| + 2.01 u (|sum x| + err)) / hw.
  eval (folded)        after non-trivial running statistics: every conv_fprop_affine output lies between the bf16
                       results of the ends of the interval acc scale + shift +- 2 (|scale| KAPPA A + u |acc scale +
                       shift|), acc the float64 conv (the rule of test_gpu_conv_epilogues.py); conv3 adds its shortcut
                       after rounding the BN output to bf16.  With DIRB200_FOLDED_EVAL=0 (a subprocess) the unfolded
                       eval sequence is checked like the training forward, without statistics.

Every training case runs three forwards on fresh inputs and parameters: eager, the one that captures the CUDA graph and
a replay (run_graphed, csrc/resnet_runner.cu).  Each must pass every check.  The whole file runs again in subprocesses
with DIRB200_SMS=7, DIRB200_GRAPH=0 and DIRB200_FUSED_STATS=0."""
import ctypes
import gc
import os
import subprocess
import sys
import time

import pytest
import torch
import torch.nn.functional as F

from test_gpu_conv import BF16_U, KAPPA
from test_gpu_conv_epilogues import candidates, chain_length, expected_rows, plan_bn
from test_gpu_layer_kernels import lanes, pool_ref, stats_nblocks, unpack_mask
from test_gpu_runner_kernels import STEM_INV, conv_table, dev_view, make_model, peek_conv

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF = torch.bfloat16
F64 = torch.float64
SLACK = 1.0 + 1e-3
EPS = float(torch.tensor(1e-5, dtype=torch.float32))
MOM = float(torch.tensor(0.1, dtype=torch.float32))
OM = float(torch.tensor(1.0, dtype=torch.float32) - torch.tensor(0.1, dtype=torch.float32))
BUDGET = 1 << 24                 # float64 elements per chunk of a reference conv

# worst measured error / bound per check kind over the file (printed with -s)
WORST = {}


def note(kind, err, bound):
    r = (err / bound.clamp_min(1e-300)).max().item() if err.numel() else 0.0
    WORST[kind] = max(WORST.get(kind, 0.0), r)


def fused_stats():
    return os.environ.get("DIRB200_FUSED_STATS", "1")[:1] != "0"


def folded_eval():
    return os.environ.get("DIRB200_FOLDED_EVAL", "1")[:1] != "0"


def lib():
    import _lib
    import _convlib, resnet  # noqa: F401
    return _lib


def peek(L, net, block, which):
    """(device pointer, rows, channels) of selector `which` (dirb200_resnet_peek)."""
    ptr, rows, ch = ctypes.c_void_p(), ctypes.c_int64(), ctypes.c_int()
    L.call("dirb200_resnet_peek", net, block, which, ctypes.byref(ptr), ctypes.byref(rows), ctypes.byref(ch))
    return ptr.value, rows.value, ch.value


def peek_bf16(L, net, block, which):
    """Zero-copy [rows, channels] bf16 view of a runner activation."""
    p, rows, c = peek(L, net, block, which)
    return dev_view(p, rows * c, "<i2").view(BF).view(rows, c)


def peek_u8(L, net, block):
    p, rows, c = peek(L, net, block, 7)
    return dev_view(p, rows * c, "|u1").view(rows, c)


def fma32(y, s, h):
    """fl32(y s + h) as fmaf forms it, for bf16 y and fp32 s, h: the product is exact in float64 (8 x 24 bits); the sum
    t = p + h is exact up to its TwoSum error e, so rounding t to fp32 is the rounding of the exact value except where t
    lies exactly halfway between two fp32 values and e != 0 breaks the tie."""
    p = y.double() * s.double()
    hd = h.double().expand_as(p)
    t = p + hd
    hv = t - p
    e = (p - (t - hv)) + (hd - hv)
    r = t.float()
    rd = r.double()
    other = torch.nextafter(r, torch.where(t > rd, torch.full_like(r, float("inf")), torch.full_like(r, -float("inf"))))
    tie = (rd != t) & ((rd + other.double()) * 0.5 == t) & (e != 0)
    up = torch.where(e > 0, torch.maximum(r, other), torch.minimum(r, other))
    return torch.where(tie, up, r)


def zbits(t):
    """bf16 bits with -0 read as +0 (fmaxf(-0, 0) may return either zero)."""
    b = t.view(torch.int16)
    return torch.where(b == -32768, torch.zeros_like(b), b)


# ------------------------------------------------------------------------------------------------ float64 convs
def conv_weight(L, net, cv):
    """The conv's own bf16 fprop operand as a float64 [cout][cin][k][k] filter (the stem: its 3x7x7 taps)."""
    block, conv, _, _, ci, co, k, _, _, _, _, stem = cv
    pk = peek_conv(L, net, block, conv)
    if stem:
        op = dev_view(pk.w_fprop, co * 256, "<i2").view(BF).view(co, 256).double()
        return op[:, torch.from_numpy(STEM_INV).to(DEV)].view(co, 3, 7, 7), pk
    return dev_view(pk.w_fprop, co * k * k * ci, "<i2").view(BF).view(co, k, k, ci).permute(0, 3, 1, 2).double(), pk


def conv64(x_nchw, w, stride, pad):
    """x float64 NCHW, w float64 [co][ci][k][k] -> [n * ho * wo, co] (NHWC rows) by a float64 GEMM."""
    n, ci, h, wd = x_nchw.shape
    co, _, k, _ = w.shape
    if k == 1 and pad == 0:
        xs = x_nchw[:, :, ::stride, ::stride]
        return xs.permute(0, 2, 3, 1).reshape(-1, ci) @ w.view(co, ci).t()
    cols = F.unfold(x_nchw, k, padding=pad, stride=stride)          # [n, ci k k, L], (ci, r, s) order
    return (cols.transpose(1, 2) @ w.reshape(co, -1).t()).reshape(-1, co)


def conv_chunks(src, n, h, w, cin, cout, k, stride, pad):
    """Yields (row slice, ref, A) over image chunks: ref = conv(x, w), A = conv(|x|, |w|), both float64.  src(b) gives
    the float64 NCHW input of images b."""
    ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    per = max(cin * k * k * ho * wo, cout * ho * wo, cin * h * w)
    step = max(1, BUDGET // per)
    for b0 in range(0, n, step):
        b1 = min(n, b0 + step)
        x = src(slice(b0, b1))
        yield slice(b0 * ho * wo, b1 * ho * wo), x, ho, wo


def conv_input(L, net, x, cv):
    """The float64-NCHW source of conv cv's input, as the reference network routes it (resnet.py Bottleneck.forward):
    the stem reads x, a block's conv1 / downsample read the previous block's output (block 0: the max-pool output),
    conv2 reads relu(bn1), conv3 relu(bn2)."""
    block, conv, _, _, ci, _, _, _, _, h, w, stem = cv
    if stem:
        xb = x.to(BF)
        return lambda b: xb[b].double()
    if conv in (0, 3):
        t = block_input(L, net, block)
    else:
        t = peek_bf16(L, net, block, 1 if conv == 1 else 3)
    assert t.shape[1] == ci, cv
    per = h * w
    return lambda b: t[b.start * per:b.stop * per].view(-1, h, w, ci).permute(0, 3, 1, 2).double()


def block_input(L, net, block):
    """The input of block `block`: the previous block's output, or the stem's max-pool output."""
    return peek_bf16(L, net, block - 1, 6) if block > 0 else peek_bf16(L, net, -1, 6)


RAW = {0: 0, 1: 2, 2: 4, 3: 5}        # conv -> peek selector of its raw output


def raw_y(L, net, cv):
    return peek_bf16(L, net, -1, 0) if cv[11] else peek_bf16(L, net, cv[0], RAW[cv[1]])


def check_conv(L, net, x, cv, n, tag):
    """y against the float64 conv, element by element; returns the conv's weight operand peek."""
    block, conv, name, _, ci, co, k, s, p, h, w, stem = cv
    wt, pk = conv_weight(L, net, cv)
    src = conv_input(L, net, x, cv)
    y = raw_y(L, net, cv)
    K = 256 if stem else k * k * ci
    for rs, xin, ho, wo in conv_chunks(src, n, h, w, ci, co, k, s, p):
        ref = conv64(xin, wt, s, p)
        A = conv64(xin.abs(), wt.abs(), s, p)
        err = (y[rs].double() - ref).abs()
        bound = BF16_U * ref.abs() + (1 + BF16_U) * KAPPA(K) * A
        note("conv y", err, bound)
        bad = ~(err <= bound)
        assert not bad.any(), (f"{tag} {name}: {int(bad.sum())} of {bad.numel()} outputs over the bound, first at row "
                               f"{rs.start + int(bad.nonzero()[0, 0])} channel {int(bad.nonzero()[0, 1])}")
        del ref, A, err, bound, xin
    return pk


# ------------------------------------------------------------------------------------------------ statistics
def channel_sums(y):
    """float64 per-channel sum y, sum y^2, sum |y| of [rows, c] bf16, in row chunks."""
    c = y.shape[1]
    s0 = torch.zeros(c, dtype=F64, device=DEV)
    s1, sa = s0.clone(), s0.clone()
    step = max(1, BUDGET // c)
    for r0 in range(0, y.shape[0], step):
        t = y[r0:r0 + step].double()
        s0 += t.sum(0)
        s1 += (t * t).sum(0)
        sa += t.abs().sum(0)
    return s0, s1, sa


def stats_chain(y, cv, n):
    """fp32 chain length of one channel sum, for the path this process takes."""
    _, _, _, _, ci, co, k, s, p, h, w, stem = cv
    rows = y.shape[0]
    if fused_stats():
        bn = plan_bn((n, h, w, ci, co, k, s, p), 0, stem)
        m_tiles = -(-rows // 128)
        n_tiles = co // bn
        return chain_length((expected_rows(m_tiles, n_tiles), n_tiles, bn, 1), m_tiles)
    nb = stats_nblocks(y, rows, co)
    return -(-rows // (nb * lanes(co))) + lanes(co) + 2


def f32(p):
    return dev_view(p, 1, "<f4")


def check_stats(L, net, m, cv, pk, y, n, rm0, rv0, tag):
    """mean / invstd / scale / shift of one BatchNorm and its running-statistics update."""
    name, pre, co = cv[2], cv[3], cv[5]
    named, bufs = dict(m.named_parameters()), dict(m.named_buffers())
    rows = float(y.shape[0])
    s0, s1, sa = channel_sums(y)
    mref = s0 / rows
    var = (s1 / rows - mref * mref).clamp_min(0)
    # sum y^2 / n - m^2 in float64 loses nothing that matters here: the variance of the stored bf16 values
    Lc = stats_chain(y, cv, n)
    dm = Lc * U * sa / rows
    dvar = Lc * U * s1 / rows + 2 * mref.abs() * dm + dm * dm
    mp, ip = ctypes.c_void_p(), ctypes.c_void_p()
    L.call("dirb200_resnet_peek_bn_stats", net, cv[0], cv[1], ctypes.byref(mp), ctypes.byref(ip))
    mean = dev_view(mp.value, co, "<f4").double()
    invstd = dev_view(ip.value, co, "<f4").double()
    r_is = 1.0 / torch.sqrt(var + EPS)
    e, b = (mean - mref).abs(), SLACK * (dm + U * mref.abs()) + 1e-30
    note("mean", e, b)
    assert (e <= b).all(), f"{tag} {name} mean: worst excess {(e - b).max().item():.3e} (L = {Lc})"
    e, b = (invstd - r_is).abs(), SLACK * r_is * (0.5 * dvar / (var + EPS) + U)
    note("invstd", e, b)
    assert (e <= b).all(), f"{tag} {name} invstd: worst relative error {(e / r_is).max().item():.3e} (L = {Lc})"
    # scale / shift from the runner's own fp32 mean, invstd and the parameters
    ga, be = named[pre + "weight"].double(), named[pre + "bias"].double()
    sc = dev_view(pk.scale, co, "<f4").double()
    sh = dev_view(pk.shift, co, "<f4").double()
    r_sc = ga * invstd
    e, b = (sc - r_sc).abs(), U * r_sc.abs() + 1e-45
    note("scale", e, b)
    assert (e <= b).all(), f"{tag} {name} scale"
    r_sh = be - mean * sc
    e, b = (sh - r_sh).abs(), U * (r_sh.abs() + (mean * sc).abs()) + 1e-45
    note("shift", e, b)
    assert (e <= b).all(), f"{tag} {name} shift"
    # running statistics, from the values before this forward
    unb = var * rows / (rows - 1)
    r_rm = OM * rm0 + MOM * mref
    r_rv = OM * rv0 + MOM * unb
    b_rm = SLACK * (MOM * dm + 4 * U * (OM * rm0.abs() + MOM * mref.abs())) + 1e-45
    b_rv = SLACK * (MOM * dvar * rows / (rows - 1) + 4 * U * (OM * rv0.abs() + MOM * unb)) + 1e-45
    e = (bufs[pre + "running_mean"].double() - r_rm).abs()
    note("running_mean", e, b_rm)
    assert (e <= b_rm).all(), f"{tag} {name} running_mean: worst excess {(e - b_rm).max().item():.3e}"
    e = (bufs[pre + "running_var"].double() - r_rv).abs()
    note("running_var", e, b_rv)
    assert (e <= b_rv).all(), f"{tag} {name} running_var: worst excess {(e - b_rv).max().item():.3e}"


# ------------------------------------------------------------------------------------------------ activations
def coeffs(pk, c):
    return dev_view(pk.scale, c, "<f4"), dev_view(pk.shift, c, "<f4")


def row_chunks(rows, c):
    step = max(1, (BUDGET // 2) // c)
    for r0 in range(0, rows, step):
        yield slice(r0, min(rows, r0 + step))


def check_act(L, net, block, conv, pk, tag):
    """relu(bn(y)) of conv1 / conv2, bit for bit."""
    y = peek_bf16(L, net, block, RAW[conv])
    a = peek_bf16(L, net, block, 1 if conv == 0 else 3)
    sc, sh = coeffs(pk, y.shape[1])
    for q in row_chunks(y.shape[0], y.shape[1]):
        ref = torch.relu(fma32(y[q], sc, sh)).to(BF)
        bad = zbits(a[q]) != zbits(ref)
        assert not bad.any(), f"{tag} block {block} a{conv + 1}: {int(bad.sum())} outputs differ"


def check_block_out(L, net, block, pk3, pkd, has_ds, with_mask, tag):
    """out = bf16(relu(fl32(y3 s3 + h3) + shortcut)) bit for bit, and its mask bits = (out > 0)."""
    y3 = peek_bf16(L, net, block, 4)
    out = peek_bf16(L, net, block, 6)
    c = y3.shape[1]
    assert c % 8 == 0
    s3, h3 = coeffs(pk3, c)
    if has_ds:
        yd = peek_bf16(L, net, block, 5)
        sd, hd = coeffs(pkd, c)
    else:
        xin = block_input(L, net, block)
        assert xin.shape == out.shape
    mask = peek_u8(L, net, block) if with_mask else None
    if with_mask:
        assert mask.shape == (out.shape[0], c // 8)
    for q in row_chunks(out.shape[0], c):
        short = fma32(yd[q], sd, hd).double() if has_ds else xin[q].double()
        ref = torch.relu((fma32(y3[q], s3, h3).double() + short).float()).to(BF)
        bad = zbits(out[q]) != zbits(ref)
        assert not bad.any(), f"{tag} block {block} output: {int(bad.sum())} outputs differ"
        if with_mask:
            bad = unpack_mask(mask[q], c) != (out[q].float() > 0)
            assert not bad.any(), f"{tag} block {block} mask: {int(bad.sum())} bits differ"


def check_pool(L, net, pk, n, h, w, tag):
    """The stem's max pool over bf16(relu(fl32(y scale + shift))) (h x w: the stem output map), values and argmax."""
    y = peek_bf16(L, net, -1, 0)
    out = peek_bf16(L, net, -1, 6)
    idx = peek_u8(L, net, -1)
    sc, sh = coeffs(pk, 64)
    hw = h * w
    assert y.shape[0] == n * hw and idx.shape == out.shape
    pw = out.shape[0] // n
    step = max(1, BUDGET // (4 * hw * 64))
    for b0 in range(0, n, step):
        b = slice(b0, min(n, b0 + step))
        act = torch.relu(fma32(y[b0 * hw:b.stop * hw], sc, sh)).to(BF).float().view(-1, h, w, 64)
        val, first = pool_ref(act)
        got = out[b0 * pw:b.stop * pw].view(val.shape)
        bad = zbits(got) != zbits(val.to(BF))
        assert not bad.any(), f"{tag} pool values: {int(bad.sum())} differ"
        bad = idx[b0 * pw:b.stop * pw].view(first.shape).long() != first
        assert not bad.any(), f"{tag} pool argmax: {int(bad.sum())} differ"


def check_encoding(L, net, enc, n, last_block, tag):
    last = peek_bf16(L, net, last_block, 6)
    c = last.shape[1]
    hw = last.shape[0] // n
    t = last.view(n, hw, c).double()
    s, sa = t.sum(1), t.abs().sum(1)
    e_sum = (hw - 1) * U * sa
    bound = SLACK * (e_sum + 2.01 * U * (s.abs() + e_sum)) / hw + 1e-45
    err = (enc.double() - s / hw).abs()
    note("encoding", err, bound)
    assert (err <= bound).all(), f"{tag} encoding: worst excess {(err - bound).max().item():.3e}"


# ------------------------------------------------------------------------------------------------ cases
CASES = [((3, 4, 6, 3), 16, 64, 64, False), ((3, 4, 6, 3), 4, 224, 224, False), ((2, 2, 1, 1), 16, 64, 64, False),
         ((3, 4, 6, 3), 1, 228, 304, True), ((3, 4, 6, 3), 8, 228, 304, True), ((3, 4, 6, 3), 256, 224, 224, False)]
IDS = ["r50_b16_64", "r50_b4_224", "shallow_b16_64", "nyud2_encoder_b1_228x304", "nyud2_encoder_b8_228x304",
       "r50_b256_224"]


def setup(layers, n, h, w):
    L = lib()
    m = make_model(layers)
    net = m._net((n, 3, h, w))
    return L, m, net, conv_table(layers, h, w)


def randomize_bn(m, table, g, running):
    """gamma in +-[0.5, 1.5] (both signs), beta ~ 0.5 N(0, 1); running statistics as well when asked."""
    named, bufs = dict(m.named_parameters()), dict(m.named_buffers())
    with torch.no_grad():
        for cv in table:
            pre, c = cv[3], cv[5]
            sgn = torch.where(torch.rand(c, generator=g, device=DEV) < 0.25, -1.0, 1.0)
            named[pre + "weight"].copy_(sgn * (0.5 + torch.rand(c, generator=g, device=DEV)))
            named[pre + "bias"].copy_(0.5 * torch.randn(c, generator=g, device=DEV))
            if running:
                bufs[pre + "running_mean"].copy_(torch.randn(c, generator=g, device=DEV))
                bufs[pre + "running_var"].copy_(0.5 + torch.rand(c, generator=g, device=DEV))


def forward(m, x, blocks, training):
    return m._run_forward_blocks(x, training=training) if blocks else m._run_forward(x, training=training)


def by_block(table):
    d = {}
    for cv in table:
        d.setdefault(cv[0], {})[cv[1]] = cv
    return d


@pytest.mark.parametrize("layers,n,h,w,blocks", CASES, ids=IDS)
def test_training_forward_in_place(layers, n, h, w, blocks):
    L, m, net, table = setup(layers, n, h, w)
    bufs = dict(m.named_buffers())
    g = torch.Generator(device=DEV).manual_seed(n + h + w + len(layers))
    blk = by_block(table)
    t0 = time.time()
    for it in range(3):                     # eager, graph capture, graph replay
        tag = f"forward {it + 1}"
        randomize_bn(m, table, g, running=(it == 0))
        x = torch.randn(n, 3, h, w, generator=g, device=DEV)
        rm0 = {cv[3]: bufs[cv[3] + "running_mean"].double().clone() for cv in table}
        rv0 = {cv[3]: bufs[cv[3] + "running_var"].double().clone() for cv in table}
        nbt0 = {cv[3]: int(bufs[cv[3] + "num_batches_tracked"]) for cv in table}
        out = forward(m, x, blocks, True)
        torch.cuda.synchronize()
        for cv in table:
            pk = check_conv(L, net, x, cv, n, tag)
            y = raw_y(L, net, cv)
            check_stats(L, net, m, cv, pk, y, n, rm0[cv[3]], rv0[cv[3]], tag)
            assert int(bufs[cv[3] + "num_batches_tracked"]) == nbt0[cv[3]] + 1, cv[3]
            if cv[11]:
                check_pool(L, net, pk, n, h // 2, w // 2, tag)
            elif cv[1] in (0, 1):
                check_act(L, net, cv[0], cv[1], pk, tag)
        for bi, convs in sorted(blk.items()):
            if bi < 0:
                continue
            pk3 = peek_conv(L, net, bi, 2)
            pkd = peek_conv(L, net, bi, 3) if 3 in convs else None
            check_block_out(L, net, bi, pk3, pkd, 3 in convs, True, tag)
        if blocks:
            ends = [sum(layers[:s + 1]) - 1 for s in range(len(layers))]
            for s, bi in enumerate(ends):
                assert torch.equal(out[s].reshape(-1), peek_bf16(L, net, bi, 6).reshape(-1)), (tag, s)
        else:
            check_encoding(L, net, out, n, sum(layers) - 1, tag)
    print(f"\ntraining forward {IDS[CASES.index((layers, n, h, w, blocks))]}: {time.time() - t0:.1f} s; worst "
          "error / bound so far: " + ", ".join(f"{k} {v:.3f}" for k, v in WORST.items()))


def check_affine(L, net, x, n, cv, shortcut, out, relu, tag):
    """One conv_fprop_affine output against the float64 conv through the eval BN affine map."""
    block, conv, name, _, ci, co, k, s, p, h, w, _ = cv
    wt, pk = conv_weight(L, net, cv)
    sc, sh = (t.double() for t in coeffs(pk, co))
    src = conv_input(L, net, x, cv)
    kap = KAPPA(k * k * ci)
    for rs, xin, ho, wo in conv_chunks(src, n, h, w, ci, co, k, s, p):
        ref = conv64(xin, wt, s, p)
        A = conv64(xin.abs(), wt.abs(), s, p)
        aff = ref * sc + sh
        err = 2 * (sc.abs() * kap * A + U * aff.abs()) + 1e-30
        got = out[rs]
        if shortcut is None:
            lo, hi = candidates(aff, err, torch.relu if relu else (lambda t: t))
        else:
            qlo, qhi = candidates(aff, err, lambda t: t)
            r = shortcut[rs].float()
            lo = torch.relu(qlo.float() + r).to(BF)
            hi = torch.relu(qhi.float() + r).to(BF)
        ok = (got >= lo) & (got <= hi)
        # reported only: |got - ref| over one bf16 rounding (two with a shortcut) plus the accumulator error
        post = torch.relu(aff) if relu and shortcut is None else aff
        if shortcut is None:
            e, b = (got.double() - post).abs(), BF16_U * post.abs() + err
        else:
            r_out = torch.relu(aff + shortcut[rs].double())
            e, b = (got.double() - r_out).abs(), BF16_U * (aff.abs() + r_out.abs()) + err
        note("eval affine", e, b)
        assert ok.all(), f"{tag} {name}: {int((~ok).sum())} of {ok.numel()} outputs outside the bound"
        del ref, A, aff, err, lo, hi


@pytest.mark.parametrize("layers,n,h,w,blocks", CASES, ids=IDS)
def test_eval_forward_in_place(layers, n, h, w, blocks):
    L, m, net, table = setup(layers, n, h, w)
    g = torch.Generator(device=DEV).manual_seed(7 * n + h + w)
    blk = by_block(table)
    x = torch.randn(n, 3, h, w, generator=g, device=DEV)
    forward(m, x, blocks, True)              # a training forward first: its masks must not be reported afterwards
    # running means ~ N(0, 1), variances in [0.5, 1.5), gammas of both signs: activations keep their magnitude through
    # the net (the extreme coefficients of test_gpu_runner_kernels.py's bn_stats_tricky overflow after a few blocks)
    randomize_bn(m, table, g, running=True)
    x = torch.randn(n, 3, h, w, generator=g, device=DEV)
    out = forward(m, x, blocks, False)
    torch.cuda.synchronize()
    tag = "eval folded" if folded_eval() else "eval unfolded"
    # the block masks belong to a training forward: refused now
    ptr, rows, ch = ctypes.c_void_p(), ctypes.c_int64(), ctypes.c_int()
    rc = L.raw("dirb200_resnet_peek")(net, 0, 7, ctypes.byref(ptr), ctypes.byref(rows), ctypes.byref(ch))
    assert rc == -1 and "not materialised" in L.last_error(), L.last_error()
    stem = table[0]
    pk = check_conv(L, net, x, stem, n, tag)
    check_pool(L, net, pk, n, h // 2, w // 2, tag)
    for bi, convs in sorted(blk.items()):
        if bi < 0:
            continue
        has_ds = 3 in convs
        if folded_eval():
            check_affine(L, net, x, n, convs[0], None, peek_bf16(L, net, bi, 1), True, tag)
            check_affine(L, net, x, n, convs[1], None, peek_bf16(L, net, bi, 3), True, tag)
            if has_ds:
                check_affine(L, net, x, n, convs[3], None, peek_bf16(L, net, bi, 5), False, tag)
                short = peek_bf16(L, net, bi, 5)
            else:
                short = block_input(L, net, bi)
            check_affine(L, net, x, n, convs[2], short, peek_bf16(L, net, bi, 6), True, tag)
        else:
            pks = {c: check_conv(L, net, x, cv, n, tag) for c, cv in convs.items()}
            check_act(L, net, bi, 0, pks[0], tag)
            check_act(L, net, bi, 1, pks[1], tag)
            check_block_out(L, net, bi, pks[2], pks.get(3), has_ds, False, tag)
    if not blocks:
        check_encoding(L, net, out, n, sum(layers) - 1, tag)
    print(f"\n{tag} {IDS[CASES.index((layers, n, h, w, blocks))]}: worst error / bound so far: " +
          ", ".join(f"{k} {v:.3f}" for k, v in WORST.items()))


# ------------------------------------------------------------------------------------------------ reruns
def rerun(env, *select, path=os.path.abspath(__file__)):
    """pytest on `path` (this file) in a fresh process with `env` added; prints its "worst" lines.  This process first
    hands its cached device memory back, so that the child has the card's memory; a failure's message starts with the
    child's own failure lines."""
    gc.collect()
    torch.cuda.empty_cache()
    e = dict(os.environ)
    e.update(env)
    t0 = time.time()
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-s", "-p", "no:cacheprovider",
                        path, *select], env=e, cwd=ROOT, capture_output=True, text=True,
                       timeout=3000)
    print(f"\n{env}: {time.time() - t0:.1f} s\n" + "\n".join(l for l in r.stdout.splitlines() if "worst" in l)[-3000:])
    why = [l for l in (r.stdout + r.stderr).splitlines() if l.startswith(("FAILED", "ERROR", "E "))]
    assert r.returncode == 0, (f"{env}: rc {r.returncode}: " + " | ".join(why[:6])[:1500] + "\n" + r.stdout[-4000:] +
                               r.stderr[-2000:])


RERUN_VARS = ("DIRB200_SMS", "DIRB200_GRAPH", "DIRB200_FUSED_STATS", "DIRB200_FOLDED_EVAL")


@pytest.mark.parametrize("env", [{"DIRB200_SMS": "7"}, {"DIRB200_GRAPH": "0"}, {"DIRB200_FUSED_STATS": "0"},
                                 {"DIRB200_FOLDED_EVAL": "0"}],
                         ids=["sms7", "no_graphs", "bn_stats_pass", "unfolded_eval"])
def test_whole_file_rerun(env):
    """This file again in a fresh process (the switches are read once per process): grids capped at 7 SMs, eager
    launches only, the separate bn_stats pass instead of the epilogue statistics; the eval test with the unfolded
    eval sequence."""
    if any(os.environ.get(k) for k in RERUN_VARS):
        pytest.skip("already a rerun")
    rerun(env, *(["-k", "eval_forward"] if "DIRB200_FOLDED_EVAL" in env else ["-k", "not rerun"]))
