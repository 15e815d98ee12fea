"""Float64 restatements of the encoder's fused glue kernels (csrc/encoder_ops.cu), the yardstick of
tests/test_encoder_ops_gpu.py.  Test infrastructure only: plain torch ops in float64 on whatever device the inputs
live on, no kernels of this package.  Each function names the reference lines it restates;
tests/test_encoder_ops_cpu.py pins them against oracle/torch_ref.py, ``F.layer_norm`` and autograd.

The case lists at the bottom are shared by the CPU and the GPU file, so that both check the same shapes and types.
"""
import math

import torch

F64 = torch.float64


# ------------------------------------------------------------------------------------------------
# LayerNorm with residual, dropout and the y + pos output (encoder.py's norms after each block)
# ------------------------------------------------------------------------------------------------
def layernorm_input(x, res=None, keep=None, p=0.0):
    """xin = dropout_p(x) + res, with the keep-mask given as a 0/1 tensor (inverted dropout: kept values / (1 - p))."""
    xin = x.to(F64)
    if keep is not None:
        xin = xin * keep.to(F64) / (1.0 - p)
    if res is not None:
        xin = xin + res.to(F64)
    return xin


def layernorm_forward(x, res, gamma, beta, eps, keep=None, p=0.0, pos=None):
    """nn.LayerNorm over the last dim of xin: biased variance, eps inside the square root.  Returns
    dict(y, y2 = y + pos, mean, rstd, xhat) in float64."""
    xin = layernorm_input(x, res, keep, p)
    mean = xin.mean(-1, keepdim=True)
    var = (xin - mean).square().mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xhat = (xin - mean) * rstd
    y = xhat * gamma.to(F64) + beta.to(F64)
    return dict(y=y, y2=None if pos is None else y + pos.to(F64), mean=mean.squeeze(-1), rstd=rstd.squeeze(-1),
                xhat=xhat)


def layernorm_backward(x, res, gamma, eps, dy, dy2=None, keep=None, p=0.0):
    """Gradients of y = LayerNorm(xin) * gamma + beta for the upstream gradient g = dy (+ dy2, the gradient of y + pos):
    d_in = rstd * (g*gamma - mean(g*gamma) - xhat * mean(g*gamma*xhat)) is the residual's gradient, dx = d_in times the
    dropout scale, dgamma = sum_rows g * xhat, dbeta = sum_rows g."""
    f = layernorm_forward(x, res, gamma, torch.zeros_like(gamma), eps, keep, p)
    xhat, rstd = f["xhat"], f["rstd"][..., None]
    g = dy.to(F64) if dy2 is None else dy.to(F64) + dy2.to(F64)
    gg = g * gamma.to(F64)
    d_in = rstd * (gg - gg.mean(-1, keepdim=True) - xhat * (gg * xhat).mean(-1, keepdim=True))
    dx = d_in if keep is None else d_in * keep.to(F64) / (1.0 - p)
    C = x.shape[-1]
    return dict(dx=dx, dres=d_in, dgamma=(g * xhat).reshape(-1, C).sum(0), dbeta=g.reshape(-1, C).sum(0),
                gg=gg, xhat=xhat, rstd=rstd.squeeze(-1))


# ------------------------------------------------------------------------------------------------
# sampling-point prep
# ------------------------------------------------------------------------------------------------
def _wh(level_hw):
    """(L, 2) [H, W] -> (L, 2) [W, H]: x offsets are divided by the level's width, y offsets by its height."""
    hw = torch.as_tensor(level_hw).to(F64)
    return torch.stack([hw[:, 1], hw[:, 0]], -1)


def tsa_prep_forward(raw, ref2d, level_hw, B, Nq, M, L, P, interleave=False):
    """temporal_self_attention.py:206-229 for num_bev_queue = 2 and L levels.  raw (B*Nq, M*2*L*P*3) holds
    [offsets (M, 2, L, P, 2) | logits (M, 2, L*P)] per query; ref2d (B*2, Nq, L, 2) is frame-major.  The softmax runs
    per (head, queue entry) over its L*P logits; loc = ref2d + offset / (W_l, H_l).  Rows come out frame-major,
    loc (B*2, Nq, M, L, P, 2), or with ``interleave`` as (B*Nq*2, M, L, P, 2), the two frames of a query adjacent."""
    LP = L * P
    r = raw.to(F64).reshape(B, Nq, -1)
    off = r[..., :M * 2 * LP * 2].reshape(B, Nq, M, 2, L, P, 2)
    att = r[..., M * 2 * LP * 2:].reshape(B, Nq, M, 2, LP).softmax(-1).reshape(B, Nq, M, 2, L, P)
    norm = _wh(level_hw).to(off.device)
    ref = ref2d.to(F64).reshape(B, 2, Nq, L, 2).permute(0, 2, 1, 3, 4)            # (B, Nq, 2, L, 2)
    loc = ref[:, :, None, :, :, None, :] + off / norm[:, None, :]                 # (B, Nq, M, 2, L, P, 2)
    if interleave:
        return (loc.permute(0, 1, 3, 2, 4, 5, 6).reshape(B * Nq * 2, M, L, P, 2),
                att.permute(0, 1, 3, 2, 4, 5).reshape(B * Nq * 2, M, L, P))
    return (loc.permute(0, 3, 1, 2, 4, 5, 6).reshape(B * 2, Nq, M, L, P, 2),
            att.permute(0, 3, 1, 2, 4, 5).reshape(B * 2, Nq, M, L, P))


def _vjp(fwd, raw, grad_loc, grad_attn):
    r = raw.detach().to(F64).requires_grad_(True)
    with torch.enable_grad():
        loc, att = fwd(r)
        loss = (loc * grad_loc.to(F64)).sum() + (att * grad_attn.to(F64)).sum()
        return torch.autograd.grad(loss, r)[0]


def tsa_prep_backward(raw, ref2d, level_hw, grad_loc, grad_attn, B, Nq, M, L, P, interleave=False):
    """d_raw of tsa_prep_forward: the softmax backward a * (ga - sum a*ga) on the logits, grad_loc / (W_l, H_l) on
    the offsets (float64 autograd of the restatement above)."""
    return _vjp(lambda r: tsa_prep_forward(r, ref2d, level_hw, B, Nq, M, L, P, interleave), raw, grad_loc, grad_attn)


def sca_prep_forward(raw, ref_cam, pair_q, pair_cam, level_hw, B, Nq, M, L, P):
    """spatial_cross_attention.py:338-372 on a (camera, query) pair list.  raw (B*Nq, M*L*P*3) holds
    [offsets (M, L, P, 2) | logits (M, L*P)] per query; ref_cam (ncam, B, Nq, D, 2).  Pair row r is query pair_q[r]
    seen by camera pair_cam[r]; rows with pair_q < 0 are padding.  The softmax runs per head over L*P logits; the
    offsets are divided by (W_l, H_l) and viewed as (P // D, D), so point p of a level adds Z-anchor p mod D.
    Returns loc (B*R, M, L, P, 2), attn (B*R, M, L, P) and the bool mask of real rows; padding rows hold NaN."""
    R, D = pair_q.numel(), ref_cam.shape[3]
    LP = L * P
    valid = pair_q.long() >= 0
    q, c = pair_q.long().clamp(min=0), pair_cam.long().clamp(min=0)
    rr = raw.to(F64).reshape(B, Nq, -1)[:, q]                                      # (B, R, width)
    norm = _wh(level_hw).to(rr.device)
    off = (rr[..., :M * LP * 2].reshape(B, R, M, L, P, 2) / norm[:, None, :]).reshape(B, R, M, L, P // D, D, 2)
    rc = ref_cam.to(F64)[c, :, q].permute(1, 0, 2, 3)                             # (B, R, D, 2)
    loc = (rc[:, :, None, None, None] + off).reshape(B, R, M, L, P, 2)
    att = rr[..., M * LP * 2:].reshape(B, R, M, LP).softmax(-1).reshape(B, R, M, L, P)
    nan = torch.tensor(float("nan"), dtype=F64, device=rr.device)
    loc = torch.where(valid[None, :, None, None, None, None], loc, nan)
    att = torch.where(valid[None, :, None, None, None], att, nan)
    return loc.reshape(B * R, M, L, P, 2), att.reshape(B * R, M, L, P), valid


def sca_prep_backward(raw, ref_cam, pair_q, pair_cam, level_hw, grad_loc, grad_attn, B, Nq, M, L, P):
    """d_raw of sca_prep_forward over the real pair rows: per query, the sum over the cameras that see it (zero for a
    query no camera sees)."""
    R = pair_q.numel()
    valid = (pair_q.long() >= 0).repeat(B)

    def fwd(r):
        loc, att, _ = sca_prep_forward(r, ref_cam, pair_q, pair_cam, level_hw, B, Nq, M, L, P)
        return loc[valid], att[valid]

    gl = grad_loc.reshape(B * R, -1)[valid].reshape(-1, M, L, P, 2)
    ga = grad_attn.reshape(B * R, -1)[valid].reshape(-1, M, L, P)
    return _vjp(fwd, raw, gl, ga)


# ------------------------------------------------------------------------------------------------
# SCA combine, reductions and elementwise
# ------------------------------------------------------------------------------------------------
def camera_count(pair_q, Nq):
    """Number of cameras that see each query, from the pair list."""
    q = pair_q.long()
    q = q[q >= 0]
    return torch.zeros(Nq, dtype=F64, device=pair_q.device).index_add_(0, q, torch.ones_like(q, dtype=F64))


def sca_combine_forward(out, pair_q, B, Nq):
    """spatial_cross_attention.py:165-172: slots[b, q] = sum of the pair rows of q / max(1, #cameras seeing q).
    out (B*R, C) -> (B, Nq, C)."""
    R, C = pair_q.numel(), out.shape[-1]
    valid = pair_q.long() >= 0
    o = out.to(F64).reshape(B, R, C)[:, valid]
    slots = torch.zeros(B, Nq, C, dtype=F64, device=out.device).index_add_(1, pair_q.long()[valid], o)
    return slots / camera_count(pair_q, Nq).clamp(min=1)[None, :, None]


def sca_combine_backward(g_slots, pair_q, B, Nq):
    """Gradient of sca_combine_forward: row r gets g_slots[b, q_r] / count(q_r); padding rows hold NaN."""
    R = pair_q.numel()
    valid = pair_q.long() >= 0
    q = pair_q.long().clamp(min=0)
    g = g_slots.to(F64)[:, q] / camera_count(pair_q, Nq).clamp(min=1)[q][None, :, None]
    g = torch.where(valid[None, :, None], g, torch.tensor(float("nan"), dtype=F64, device=g.device))
    return g.reshape(B * R, -1)


def colsum(x, out0=None):
    """out0 + sum over rows of x (rows, C), and sum over rows of |x| (the scale of the reduction's rounding)."""
    s = x.to(F64).sum(0)
    a = x.to(F64).abs().sum(0)
    if out0 is not None:
        s, a = s + out0.to(F64), a + out0.to(F64).abs()
    return s, a


def sum_tensors(ts):
    """Elementwise sum of the tensors, and the sum of their magnitudes."""
    s = sum(t.to(F64) for t in ts)
    a = sum(t.to(F64).abs() for t in ts)
    return s, a


def dropout_scale32(p):
    """The inverted-dropout scale 1 / (1 - p), rounded once to fp32."""
    return float(torch.tensor(1.0 / (1.0 - float(torch.tensor(p, dtype=torch.float32))), dtype=torch.float32))


def dropout_kept(x, scale32):
    """Value of a kept element of dropout(x): x * scale with the product rounded to fp32, then to x's storage type."""
    return (x.to(F64) * scale32).to(torch.float32).to(x.dtype)


def relu_dropout_backward(dy, h, scale32):
    """Gradient w.r.t. z of h = dropout_p(relu(z)) from h alone: dy * scale where h != 0, else 0; the product rounded
    to fp32, then to storage."""
    return torch.where(h != 0, (dy.to(F64) * scale32).to(torch.float32).to(dy.dtype), torch.zeros_like(dy))


# ------------------------------------------------------------------------------------------------
# rounding units (the bars of the GPU tests are stated in these)
# ------------------------------------------------------------------------------------------------
U32 = 2.0 ** -24                       # unit roundoff of fp32


def ulp(ref, dtype):
    """One storage ulp of ``dtype`` at |ref| (float64); the subnormal spacing below the normal range."""
    mant = {torch.float32: 23, torch.bfloat16: 7, torch.float16: 10}[dtype]
    emin = {torch.float32: -126, torch.bfloat16: -126, torch.float16: -14}[dtype]
    a = ref.abs().clamp(min=2.0 ** emin)
    return torch.exp2(torch.floor(torch.log2(a)) - mant)


# ------------------------------------------------------------------------------------------------
# cases shared by tests/test_encoder_ops_cpu.py and tests/test_encoder_ops_gpu.py
# ------------------------------------------------------------------------------------------------
H100_SMS = 132                         # stand-in for multi_processor_count where no device is present

# (activation, parameter) storage pairs the LayerNorm kernels are instantiated for
LN_DTYPES = [("float32", "float32"), ("bfloat16", "float32"), ("bfloat16", "bfloat16"), ("float16", "float32"),
             ("float16", "float16")]
# rows: ends inside a warp's 4-row group (1, 3, 5, 31, 33), whole groups (4, 32), one row past a chunk of the
# backward's grid ("chunk+1", resolved from the SM count by ln_rows), and a large count
LN_ROWS = [1, 3, 4, 5, 31, 32, 33, "chunk+1", 40000]
# (residual, pos output, twin output, strided dy2, dropout p, eps); strided = dy2 is a column slice of a wider
# gradient (ld2 = 2C); pos without strided = contiguous dy2
LN_MODES = [
    dict(res=True, pos=True, twin=False, strided=True, p=0.0, eps=1e-5),
    dict(res=True, pos=False, twin=False, strided=False, p=0.3, eps=1e-5),
    dict(res=False, pos=False, twin=False, strided=False, p=0.0, eps=1e-1),
    dict(res=True, pos=False, twin=True, strided=False, p=0.3, eps=1e-5),
    dict(res=False, pos=True, twin=False, strided=False, p=0.3, eps=1e-1),
]


def ln_cases():
    """Every (C, dtype pair) at every row count; the modes rotate so that each one meets every row count and every
    dtype pair.  Two extra data kinds: rows that are constant (variance 0) and rows of 1000 + N(0, 1) (fp32)."""
    out = []
    for C in (256, 512):
        for di, (adt, pdt) in enumerate(LN_DTYPES):
            for ri, rows in enumerate(LN_ROWS):
                mi = (ri + di + (C == 512)) % len(LN_MODES)
                out.append(dict(C=C, adt=adt, pdt=pdt, rows=rows, data="randn", **LN_MODES[mi]))
        out.append(dict(C=C, adt="float32", pdt="float32", rows=37, data="const", **LN_MODES[0]))
        out.append(dict(C=C, adt="bfloat16", pdt="bfloat16", rows=37, data="const", **LN_MODES[2]))
        out.append(dict(C=C, adt="float32", pdt="float32", rows=300, data="offset", **LN_MODES[2]))
        out.append(dict(C=C, adt="float32", pdt="float32", rows=300, data="offset", **LN_MODES[1]))
    return out


def ln_case_id(c):
    m = "".join(k for k in ("res", "pos", "twin", "strided") if c[k])
    return f"C{c['C']}-{c['adt']}-{c['pdt']}-rows{c['rows']}-{c['data']}-{m or 'plain'}-p{c['p']}-eps{c['eps']}"


def ln_rows(rows, sms):
    """Resolve "chunk+1": the backward gives each CTA ceil(rows / (4 * SMs)) rows rounded up to 8; 16 * (4*SMs - 1) + 1
    rows make that 16, and the last of the 4*SMs CTAs gets exactly one row."""
    return 16 * (4 * sms - 1) + 1 if rows == "chunk+1" else rows


# TSA prep: (M, L, P, interleave, B, Nq, d_raw dtype).  M = 8 with L*P in {2, 4, 8, 16, 32} runs tsa_prep_m8<L*P/2>;
# anything else runs the generic kernels (frame-major rows only).
def tsa_cases():
    dts = ["float32", "bfloat16", "float16"]
    out = []
    for i, (L, P) in enumerate([(1, 2), (2, 1), (1, 4), (2, 2), (2, 4), (4, 4), (4, 8), (2, 16)]):
        for il in (0, 1):
            out.append(dict(M=8, L=L, P=P, interleave=il, B=1 + 2 * ((i + il) % 2), Nq=37 + 13 * il,
                            dt=dts[(i + il) % 3]))
    for i, (M, L, P) in enumerate([(4, 3, 4), (6, 3, 4), (8, 3, 4), (6, 1, 4)]):
        for j, dt in enumerate(dts):
            out.append(dict(M=M, L=L, P=P, interleave=0, B=1 + 2 * ((i + j) % 2), Nq=29, dt=dt))
    return out


def tsa_case_id(c):
    return f"M{c['M']}-L{c['L']}-P{c['P']}-il{c['interleave']}-B{c['B']}-Nq{c['Nq']}-{c['dt']}"


# SCA prep: (M, L, P, D, ncam, B, Nq, d_raw dtype).  M = 8 with L*P in {4, 8, 16, 32, 64} runs sca_prep_*_m8<L*P/4>;
# anything else the generic kernels.  ncam > 8 crosses the camera batch of sca_prep_bwd_m8.
def sca_cases():
    dts = ["float32", "bfloat16", "float16"]
    out = []
    shapes = [(1, 4, 1), (1, 4, 4), (2, 4, 2), (4, 4, 4), (4, 8, 4), (4, 8, 2), (4, 16, 4), (2, 32, 1)]
    for i, (L, P, D) in enumerate(shapes):
        for j, dt in enumerate(dts):
            out.append(dict(M=8, L=L, P=P, D=D, ncam=(6, 12, 16)[(i + j) % 3], B=1 + 2 * ((i + j) % 2),
                            Nq=45 + 4 * j, dt=dt))
    for i, (M, L, P, D) in enumerate([(4, 4, 8, 4), (8, 3, 4, 2), (6, 2, 4, 1)]):
        for j, dt in enumerate(dts):
            out.append(dict(M=M, L=L, P=P, D=D, ncam=(6, 16, 12)[(i + j) % 3], B=1 + 2 * ((i + j) % 2), Nq=37,
                            dt=dt))
    return out


def sca_case_id(c):
    return f"M{c['M']}-L{c['L']}-P{c['P']}-D{c['D']}-cams{c['ncam']}-B{c['B']}-Nq{c['Nq']}-{c['dt']}"


# level shapes (H, W), all with H != W
LEVEL_HW = [(23, 41), (12, 21), (6, 11), (3, 5)] * 4


def make_pairs(Nq, ncam, seed, pad=5):
    """A hand-built pair list: query q is seen by 0, 1, 2, all ncam or 3 cameras (q mod 5), on cameras drawn at
    random; rows are camera-major like ScaPlan's, followed by ``pad`` padding rows (pair_q = pair_cam = -1).
    Returns pair_q, pair_cam (R,) int32 and pair_of (ncam, Nq) int32 = row or -1, on the CPU."""
    g = torch.Generator().manual_seed(seed)
    seen = torch.zeros(ncam, Nq, dtype=torch.bool)
    for q in range(Nq):
        n = (0, 1, 2, ncam, min(3, ncam))[q % 5]
        seen[torch.randperm(ncam, generator=g)[:n], q] = True
    pq, pc = [], []
    pair_of = torch.full((ncam, Nq), -1, dtype=torch.int32)
    for c in range(ncam):
        for q in seen[c].nonzero().flatten().tolist():
            pair_of[c, q] = len(pq)
            pq.append(q)
            pc.append(c)
    pq += [-1] * pad
    pc += [-1] * pad
    return torch.tensor(pq, dtype=torch.int32), torch.tensor(pc, dtype=torch.int32), pair_of


# colsum: C in {8, 48, 192, 256, 768, 1024 (largest fp32 width), 2048 (largest 16-bit width)}; rows around one CTA's
# 64-row minimum, one row past a CTA boundary ("cta+1", resolved by colsum_rows), and 185000 (a real bias-gradient
# height) at the head widths.
COLSUM_C = [8, 48, 192, 256, 768, 1024, 2048]
COLSUM_ROWS = [1, 63, 64, 65, "cta+1"]


def colsum_cases():
    out = []
    for i, C in enumerate(COLSUM_C):
        dts = ["float32", "bfloat16", "float16"] if C <= 1024 else ["bfloat16", "float16"]
        for j, rows in enumerate(COLSUM_ROWS):
            out.append(dict(C=C, rows=rows, dt=dts[(i + j) % len(dts)], det=bool((i + j) % 2), acc=bool(j % 2)))
    for C, dt, det in ((192, "float32", False), (768, "bfloat16", True), (2048, "float16", False)):
        out.append(dict(C=C, rows=185000, dt=dt, det=det, acc=True))
    return out


def colsum_case_id(c):
    return f"C{c['C']}-rows{c['rows']}-{c['dt']}-{'det' if c['det'] else 'atomic'}{'-acc' if c['acc'] else ''}"


def colsum_rows(rows, sms):
    """Resolve "cta+1": colsum gives each CTA max(64, ceil(rows / (4 * SMs))) rows; 100 * (4*SMs - 1) + 1 rows make
    that 100, and the last of the 4*SMs CTAs gets exactly one row."""
    return 100 * (4 * sms - 1) + 1 if rows == "cta+1" else rows


def colsum_plan(rows, sms):
    """(rows per CTA, CTAs) of colsum's launch."""
    rpc = max(64, -(-rows // (4 * sms)))
    return rpc, -(-rows // rpc)


# sum_tensors: n = 1..8 in each dtype; element counts with a partial last CTA (256 threads x one 16 B vector each), one
# vector only, and one large enough for the grid-stride loop (grid capped at 16 CTAs per SM)
def sum_cases():
    out = []
    for n in range(1, 9):
        for j, dt in enumerate(["float32", "bfloat16", "float16"]):
            vec = 4 if dt == "float32" else 8
            numel = (vec, vec * (256 * 3 + 5), vec * (256 * 16 * 140 + 77))[(n + j) % 3]
            out.append(dict(n=n, dt=dt, numel=numel))
    return out


def sum_case_id(c):
    return f"n{c['n']}-{c['dt']}-numel{c['numel']}"


# dropout_inplace / relu_dropout_backward: element counts with a partial last CTA, p in {0.1, 0.3, 0.5}
def dropout_cases():
    out = []
    for j, dt in enumerate(["float32", "bfloat16", "float16"]):
        vec = 4 if dt == "float32" else 8
        for k, p in enumerate((0.1, 0.3, 0.5)):
            out.append(dict(dt=dt, p=p, numel=vec * (256 * (200 + 37 * k) + 3 + j)))
    return out


def dropout_case_id(c):
    return f"{c['dt']}-p{c['p']}-numel{c['numel']}"


# SCA combine: each dtype at C in {256, 32} (C a multiple of 8), 6 / 12 / 16 cameras, B in {1, 3}
def combine_cases():
    out = []
    for j, dt in enumerate(["float32", "bfloat16", "float16"]):
        for k, C in enumerate((256, 32)):
            out.append(dict(dt=dt, C=C, ncam=(6, 12, 16)[(j + k) % 3], B=1 + 2 * ((j + k) % 2), Nq=53))
    return out


def combine_case_id(c):
    return f"{c['dt']}-C{c['C']}-cams{c['ncam']}-B{c['B']}"


def binomial_bound(n, p, sigmas=6.0):
    """sigmas standard deviations of the number of successes of n Bernoulli(p) trials."""
    return sigmas * math.sqrt(n * p * (1.0 - p))
