"""Float64 restatement of the wgmma projection GEMMs (csrc/gemm.cu), the yardstick of tests/test_gemm_fp64_gpu.py.
Test infrastructure only: plain torch ops on whatever device the inputs live on, no kernels of this package.
tests/test_gemm_fp64_cpu.py pins it against integer arithmetic and shows that it rejects plausible kernel bugs.

Arithmetic (the header comment of gemm.cu):

    forward  Y  = act(X W^T + bias) (+ addend)        ReLU before the addend
    dgrad    dX = dY W (+ addend)
    wgrad    dW = dY^T X,  db = colsum(dY);  the accumulate-into form dW += dY^T X, db += colsum(dY)

The host plans (``ws_block``, ``wgrad_plan`` and the CTA partition of the weight-stationary kernel) are restated for a
given SM count, so every case declares up front which instantiation it must launch, its column block, its split count,
rows per split and workspace size.

Two input regimes, because each catches what the other cannot:

1. Exact regime.  Operands are integers in [-4, 4] times a power of two; bias and addend are dyadic values of a few
   bits.  The generator asserts that every partial sum of |products| along the reduction stays below 2^22 product
   quanta, so no float32 operation in any accumulation order rounds: the fp32 accumulation, bias, ReLU, addend, the
   split reductions and the two-pass slab sums are all exact, and the output must equal RN_out(y64) bit for bit
   (16-bit outputs via fp32(y64), which is exact, then torch's round-to-nearest-even).  This regime sees coverage and
   indexing bugs at any M -- a dropped row, a duplicated k-block, a wrong column block or split stride, db missing a
   split -- because there is no rounding error for them to hide in.  Deliberate extras: ties at the 16-bit rounding
   point (round-half-to-even), fp16 results >= 65520 (must become +-inf) and fp16 results in the subnormal range.
2. Rounding regime.  Random normals at realistic scales, compared per element against a bar built from the
   magnitudes the restatement returns (sum_k |a_k b_k|, |bias|, |addend|, |y64|), one ``bar_*`` function per
   arithmetic path.  This regime checks the rounding itself (accumulation length, double rounding, the 16-bit
   conversion) on data where exact arithmetic is impossible.  Its bars grow with M: at M = 184950 one dropped
   reduction row (an error of about 1) fits inside them, which is why the exact regime exists.

Assumption behind every accumulation bar: the tensor cores' fp32 accumulation of bf16 / fp16 products rounds at most
once per k16 step (the 16 products of one wgmma k-step and the running sum combine with one rounding, error <= u |sum|).
Nobody has measured this on Hopper; the GPU file reports the worst err / bar of every case so that a path close to 1
shows.  With that, n successive rounded steps cost gamma_n * sum |a b| (Higham, Lemma 3.1), with n = k16 steps of the
longest split + the split reductions + the epilogue additions.
"""
import math

import torch

F64 = torch.float64
U32 = 2.0 ** -24
UNIT = {torch.float32: U32, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
# half the spacing of the subnormals: the absolute rounding error of a store below the normal range
TINY = {torch.float32: 2.0 ** -150, torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -134}
TE = {torch.bfloat16: "__nv_bfloat16", torch.float16: "__half"}
CNAME = {torch.bfloat16: "__nv_bfloat16", torch.float16: "__half", torch.float32: "float"}
EXACT_LIMIT = 2 ** 22

KBM, KBK, KWS_ROWS, KWS_WEIGHT_MAX = 128, 64, 64, 128 * 1024

MUTATIONS = ("kblock_partial_16", "double_rounding", "truncate_store", "bias_partner", "relu_after_addend",
             "drop_last_row", "db_missing_split", "slabs_16bit")


def gamma(n, u=U32):
    """gamma_n = n u / (1 - n u): the relative bound of n successive roundings (Higham, Lemma 3.1)."""
    return n * u / (1.0 - n * u)


# ------------------------------------------------------------------------------------------------
# host plans (gemm.cu: ws_block, launch_ws, wgrad_plan, bevf_linear_wgrad_workspace_bytes)
# ------------------------------------------------------------------------------------------------
def ws_block(N, R):
    """Column block of the weight-stationary kernel for N output columns and reduction R; 0: streamed kernel."""
    bn = 256
    while bn > 64 and (bn * R * 2 > KWS_WEIGHT_MAX or bn // 2 >= N):
        bn //= 2
    return bn if bn * R * 2 <= KWS_WEIGHT_MAX else 0


def ws_partition(M, N, bn, sms):
    """(tiles_m, tiles_n, groups) of launch_ws: CTA g * tiles_n + j owns row tiles [g T / G, (g + 1) T / G)."""
    tiles_m, tiles_n = -(-M // KWS_ROWS), -(-N // bn)
    return tiles_m, tiles_n, max(1, min(sms // tiles_n, tiles_m))


def wgrad_plan(M, N, K, sms):
    bn = 128 if K % 128 == 0 else 64
    tiles_m = -(-N // KBM)
    splits = -(-sms // (tiles_m * (K // bn)))
    rows = -(-M // splits)
    rows = -(-rows // 64) * 64
    splits = -(-M // rows)
    return dict(bn=bn, splits=splits, rows=rows, n_pad=tiles_m * KBM)


def workspace_bytes(M, N, K, sms):
    if M <= 0 or N <= 0 or K <= 0 or K % 64:
        return 0
    p = wgrad_plan(M, N, K, sms)
    return p["splits"] * p["n_pad"] * (K + 1) * 4 + 256


def plan(case, sms):
    """What the case must launch: kernel name prefixes (``kernels``), BN, and the split / partition numbers."""
    op, M, N, K, dt = case["op"], case["M"], case["N"], case["K"], case["dtype"]
    te = TE[dt]
    if op in ("fwd", "dgrad"):
        # forward: N output columns, reduction K; dgrad: K output columns, reduction N
        cols, red = (N, K) if op == "fwd" else (K, N)
        bn = ws_block(cols, red)
        if bn:
            tiles_m, tiles_n, groups = ws_partition(M, cols, bn, sms)
            return dict(kernels=(f"gemm_ws_wgmma<{bn}, {str(op == 'dgrad').lower()}, {te}>",), bn=bn, ws=True,
                        tiles_m=tiles_m, tiles_n=tiles_n, groups=groups, steps=red // 16)
        bn = (128 if N > 64 else 64) if op == "fwd" else (128 if K % 128 == 0 else 64)
        return dict(kernels=(f"gemm_bf16_wgmma<{bn}, false, {str(op == 'dgrad').lower()}, {te}>",), bn=bn, ws=False,
                    steps=red // 16)
    p = wgrad_plan(M, N, K, sms)
    ks = [f"gemm_bf16_wgmma<{p['bn']}, true, true, {te}>"]
    if op == "wgrad_out":
        ks.append(f"wgrad_reduce_kernel<{CNAME[case['grad_dtype']]}, false>")
    elif op == "wgrad_into":
        ks.append("wgrad_reduce_kernel<float, true>")
    p.update(kernels=tuple(ks), steps=p["rows"] // 16, last_rows=M - (p["splits"] - 1) * p["rows"],
             workspace=workspace_bytes(M, N, K, sms) if op != "wgrad" else 0)
    return p


# ------------------------------------------------------------------------------------------------
# rounding helpers
# ------------------------------------------------------------------------------------------------
def rn(v64, dtype):
    """Round-to-nearest-even of float64 values to ``dtype`` via fp32 (exact in the exact regime), as float64."""
    return v64.to(torch.float32).to(dtype).to(F64)


def rz16(v64, dtype):
    """Round-toward-zero to a 16-bit type (a truncating store): where RN stepped away from zero, the 16-bit pattern
    one below (sign-magnitude: one unit less in magnitude; +-inf becomes the largest finite value)."""
    f = v64.to(torch.float32)
    r = f.to(dtype)
    away = r.to(F64).abs() > f.to(F64).abs()
    return torch.where(away, (r.view(torch.int16) - 1).view(dtype), r).to(F64)


def is_tie(y64, dtype):
    """y64 lies exactly halfway between two adjacent values of ``dtype``."""
    r = y64.to(torch.float32).to(dtype).to(F64)
    other = 2 * y64 - r
    return (r != y64) & torch.isfinite(r) & (other.to(torch.float32).to(dtype).to(F64) == other) & (other != r)


# ------------------------------------------------------------------------------------------------
# the restatement
# ------------------------------------------------------------------------------------------------
def _blocked(a, b, block, out_dtype):
    """a (M, R) @ b (R, N) with every 64-long reduction block's partial sum rounded to ``out_dtype``."""
    acc = torch.zeros(a.shape[0], b.shape[1], dtype=F64, device=a.device)
    for r0 in range(0, a.shape[1], block):
        acc += rn(a[:, r0:r0 + block] @ b[r0:r0 + block], out_dtype)
    return acc


def forward(x, w, bias=None, addend=None, relu=False, out_dtype=torch.float32, mutate=None):
    """Y = act(X W^T + bias) (+ addend) in float64.  Returns dict(y: the float64 value, want: the value the kernel
    must store (RN to out_dtype; float64), mag: sum_k |x w| + |bias| + |addend|, pre: the pre-addend value)."""
    x64, w64 = x.to(F64), w.to(F64)
    if mutate == "kblock_partial_16":
        acc = _blocked(x64, w64.t(), KBK, torch.bfloat16 if out_dtype == torch.float32 else out_dtype)
    else:
        acc = x64 @ w64.t()
    mag = x64.abs() @ w64.abs().t()
    if bias is not None:
        b = bias.to(F64)
        if mutate == "bias_partner":
            b = b.view(-1, 2).flip(1).reshape(-1)
        acc = acc + b
        mag = mag + bias.to(F64).abs()
    pre = acc
    if relu and mutate != "relu_after_addend":
        pre = pre.clamp(min=0)
    y = pre
    if addend is not None:
        a = addend.to(F64)
        y = (rn(pre, out_dtype) if mutate == "double_rounding" else pre) + a
        mag = mag + a.abs()
    if relu and mutate == "relu_after_addend":
        y = y.clamp(min=0)
    want = rz16(y, out_dtype) if (mutate == "truncate_store" and out_dtype != torch.float32) else rn(y, out_dtype)
    return dict(y=y, want=want, mag=mag, pre=pre)


def dgrad(dy, w, addend=None, mutate=None):
    """dX = dY W (+ addend); the output is in the operand type."""
    return forward(dy, w.t(), addend=addend, out_dtype=dy.dtype, mutate=mutate)


def wgrad(dy, x, splits_rows, with_db=True, grad_dtype=torch.float32, dw0=None, db0=None, mutate=None):
    """dW = dY^T X, db = colsum(dY) (+ dw0 / db0 for the accumulate-into form) in float64, with the split structure
    ``splits_rows`` = (splits, rows) for the mutations that need it.  Returns dict(dw, db: float64 values, want_dw /
    want_db: what the kernel must store in grad_dtype, mag_dw / mag_db)."""
    dy64, x64 = dy.to(F64), x.to(F64)
    splits, rows = splits_rows
    M = dy.shape[0]
    if mutate == "drop_last_row":
        dy64 = dy64[:M - 1]
        x64 = x64[:M - 1]
    if mutate == "slabs_16bit":
        dw = torch.zeros(dy.shape[1], x.shape[1], dtype=F64, device=dy.device)
        db = torch.zeros(dy.shape[1], dtype=F64, device=dy.device)
        for s in range(splits):
            sl = slice(s * rows, min(M, (s + 1) * rows))
            dw = rn(dw + rn(dy64[sl].t() @ x64[sl], grad_dtype), grad_dtype)
            db = rn(db + rn(dy64[sl].sum(0), grad_dtype), grad_dtype)
    else:
        dw = dy64.t() @ x64
        if mutate == "db_missing_split" and splits > 1:
            db = dy64[:(splits - 1) * rows].sum(0)
        else:
            db = dy64.sum(0)
    mag_dw = dy.to(F64).abs().t() @ x.to(F64).abs()
    mag_db = dy.to(F64).abs().sum(0)
    if dw0 is not None:
        dw = dw + dw0.to(F64)
        mag_dw = mag_dw + dw0.to(F64).abs()
    if db0 is not None:
        db = db + db0.to(F64)
        mag_db = mag_db + db0.to(F64).abs()
    return dict(dw=dw, db=db if with_db else None, want_dw=rn(dw, grad_dtype),
                want_db=rn(db, grad_dtype) if with_db else None, mag_dw=mag_dw, mag_db=mag_db)


# ------------------------------------------------------------------------------------------------
# bars of the rounding regime, one per arithmetic path
# ------------------------------------------------------------------------------------------------
def bar_f32(mag, steps, adds=2):
    """fp32 output of the forward / dgrad: ``steps`` k16 accumulation steps (one rounding each), then the bias and the
    addend additions (``adds``), each rounding once relative to its result; ReLU does not widen an error.  Every
    intermediate is bounded by ``mag`` = sum |x w| + |bias| + |addend|, so |err| <= gamma_{steps + adds} mag."""
    return gamma(steps + adds) * mag


def bar_16(mag, y, steps, dtype, adds=2):
    """16-bit output: the fp32 value v carries e = bar_f32; the store rounds once more: |RN(v) - y| <= u16 |v| +
    TINY + e <= u16 |y| + (1 + u16) e + TINY (TINY: half a subnormal spacing, below the normal range)."""
    e = bar_f32(mag, steps, adds)
    return UNIT[dtype] * y.abs() + (1 + UNIT[dtype]) * e + TINY[dtype]


def bar_wgrad_red(mag, steps, splits):
    """fp32 dW by red.add across splits: every split's partial tile carries gamma_steps of its own magnitudes, and the
    splits reduce into dW (which starts at zero) in any order: splits more roundings."""
    return gamma(steps + splits) * mag


def bar_wgrad_two_pass(mag, y, steps, splits, dtype):
    """Two-pass dW: per-split slabs (gamma_steps), summed in fp32 in split order (splits - 1 additions), converted once
    to ``dtype`` (nothing for fp32)."""
    e = gamma(steps + splits) * mag
    if dtype == torch.float32:
        return e
    return UNIT[dtype] * y.abs() + (1 + UNIT[dtype]) * e + TINY[dtype]


def bar_accumulate_into(mag, steps, splits):
    """dW += slab sum (deterministic mode): the two-pass fp32 sum plus one addition into the old value; ``mag``
    includes |dW_old|."""
    return gamma(steps + splits + 1) * mag


def db_steps(rows):
    """Column sums of dY: a lane adds every fourth row of its split serially (rows / 4), then two shuffles."""
    return rows // 4 + 2


# ------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------
def _ints(gen, shape, device, lo=-4, hi=4):
    return torch.randint(lo, hi + 1, shape, generator=gen, device=device, dtype=torch.int8).to(torch.float32)


def check_exact_bound(a_abs, b_abs):
    """Every partial sum of |products| of a (M, R) @ b (R, N), in product quanta, stays below 2^22, so that no fp32
    operation of any accumulation order rounds.  (max_m sum_k |a_mk|) * max|b| bounds every partial sum."""
    bound = a_abs.sum(1).max().item() * b_abs.max().item()
    assert bound < EXACT_LIMIT, f"exact regime: partial sums may reach {bound} >= 2^22 quanta"
    return bound


def make_inputs(case, device="cpu"):
    """Storage-typed inputs of a case (see ``cases``), drawn from a generator on ``device`` (CPU for every case the
    mutation checks revisit, so both files see the same numbers)."""
    op, M, N, K, dt = case["op"], case["M"], case["N"], case["K"], case["dtype"]
    gdev = "cpu" if case.get("cpu_gen", True) else device
    g = torch.Generator(device=gdev).manual_seed(case["seed"])
    exact = case["regime"] == "exact"
    special = case.get("special")
    # operand shapes: (a, b) with the product a @ b^T for fwd, a @ b for dgrad, a^T @ b for wgrad
    if op == "fwd":
        sa, sb = (M, K), (N, K)
    elif op == "dgrad":
        sa, sb = (M, N), (N, K)
    else:
        sa, sb = (M, N), (M, K)
    ea, eb = 0, 0
    if special == "subnormal":
        ea, eb = -11, -14
    if exact:
        a = _ints(g, sa, gdev) * 2.0 ** ea
        b = _ints(g, sb, gdev) * 2.0 ** eb
        ia, ib = (a * 2.0 ** -ea).abs(), (b * 2.0 ** -eb).abs()
        if op == "fwd":
            check_exact_bound(ia, ib.t())
        elif op == "dgrad":
            check_exact_bound(ia, ib)
        else:
            check_exact_bound(ia.t(), ib)
    else:
        a = torch.randn(sa, generator=g, device=gdev, dtype=torch.float32)
        b = torch.randn(sb, generator=g, device=gdev, dtype=torch.float32)
        if op in ("fwd", "dgrad"):
            b = b / math.sqrt(sb[1] if op == "fwd" else sb[0])
    out = dict(a=a.to(dt).to(device), b=b.to(dt).to(device))
    q = 2.0 ** (ea + eb)
    cols = N if op == "fwd" else K
    if case.get("bias"):
        bdt = torch.float32 if case["bias"] == "f32" else dt
        if exact:
            bias = _ints(g, (cols,), gdev, -64, 64) * q
            if special == "ties":
                bias = bias + (256.0 if dt == torch.bfloat16 else 2048.0) * q
            if special == "inf":
                bias = torch.where(torch.arange(cols, device=gdev) % 2 == 0, 65504.0, -65504.0).to(F64)
        else:
            bias = torch.randn(cols, generator=g, device=gdev, dtype=torch.float32)
        out["bias"] = bias.to(bdt).to(device)
    if case.get("addend"):
        if exact:
            add = _ints(g, (M, cols), gdev, -32, 32) * (q * 0.5)
            if special == "ties":
                add = add + (256.0 if dt == torch.bfloat16 else 2048.0) * q
        else:
            add = torch.randn((M, cols), generator=g, device=gdev, dtype=torch.float32)
        out["addend"] = add.to(dt).to(device)
    if op == "wgrad_into":
        init = _ints(g, (N, K), gdev, -64, 64) if exact else torch.randn((N, K), generator=g, device=gdev) * 10
        out["dw0"] = init.to(torch.float32).to(device)
        out["db0"] = (_ints(g, (N,), gdev, -64, 64) if exact else torch.randn(N, generator=g, device=gdev)).to(
            torch.float32).to(device)
    for name, idx, value in case.get("poison", ()):
        out[name][idx] = value
    return out


def reference(case, inp, sms, mutate=None):
    """The restatement of ``case`` on inputs ``inp``: dict of (name -> (want, bar or None)) per output, float64."""
    op, dt = case["op"], case["dtype"]
    pl = plan(case, sms)
    res = {}
    if op == "fwd":
        odt = torch.float32 if case.get("out") == "f32" else dt
        r = forward(inp["a"], inp["b"], inp.get("bias"), inp.get("addend"), case.get("relu", False), odt, mutate)
        adds = int("bias" in inp) + int("addend" in inp)
        bar = bar_f32(r["mag"], pl["steps"], adds) if odt == torch.float32 else bar_16(r["mag"], r["y"], pl["steps"],
                                                                                      odt, adds)
        res["y"] = (r["want"], r["y"], bar)
    elif op == "dgrad":
        r = dgrad(inp["a"], inp["b"], inp.get("addend"), mutate)
        adds = int("addend" in inp)
        res["y"] = (r["want"], r["y"], bar_16(r["mag"], r["y"], pl["steps"], dt, adds))
    else:
        gdt = case.get("grad_dtype", torch.float32)
        r = wgrad(inp["a"], inp["b"], (pl["splits"], pl["rows"]), case.get("db", False), gdt, inp.get("dw0"),
                  inp.get("db0"), mutate)
        s, st, sd = pl["splits"], pl["steps"], db_steps(pl["rows"])
        if op == "wgrad":
            bw, bb = bar_wgrad_red(r["mag_dw"], st, s), bar_wgrad_red(r["mag_db"], sd, s)
        elif op == "wgrad_out":
            bw = bar_wgrad_two_pass(r["mag_dw"], r["dw"], st, s, gdt)
            bb = bar_wgrad_two_pass(r["mag_db"], r["db"], sd, s, gdt) if r["db"] is not None else None
        else:
            bw, bb = bar_accumulate_into(r["mag_dw"], st, s), bar_accumulate_into(r["mag_db"], sd, s)
        res["dw"] = (r["want_dw"], r["dw"], bw)
        if r["db"] is not None:
            res["db"] = (r["want_db"], r["db"], bb)
    return res


# ------------------------------------------------------------------------------------------------
# the cases of tests/test_gemm_fp64_gpu.py
# ------------------------------------------------------------------------------------------------
_DTN = {torch.bfloat16: "bf16", torch.float16: "f16", torch.float32: "f32"}


def case_id(c):
    tags = [c["op"], _DTN[c["dtype"]], c["regime"], f"{c['M']}x{c['N']}x{c['K']}"]
    if c.get("bias"):
        tags.append("b" + c["bias"])
    tags += [t for t in ("relu", "addend", "db") if c.get(t)]
    if c.get("out") == "f32":
        tags.append("of32")
    if "grad_dtype" in c:
        tags.append("g" + _DTN[c["grad_dtype"]])
    if c.get("special"):
        tags.append(c["special"])
    if c.get("poison"):
        tags.append("poison")
    return "-".join(tags)


def cases(sms):
    """Every case of the GPU file, for a device with ``sms`` SMs (the CTA-partition edges depend on it).  Each is a
    dict: family (one child process per family and dtype), op, M, N, K, dtype, regime, options, seed, id."""
    out = []

    def add(family, op, M, N, K, regimes=("exact", "round"), dtypes=(torch.bfloat16, torch.float16), **kw):
        for dt in dtypes:
            for rg in regimes:
                c = dict(family=family, op=op, M=M, N=N, K=K, dtype=dt, regime=rg, **kw)
                c["id"] = case_id(c)
                c["seed"] = sum(ord(ch) * (i + 1) for i, ch in enumerate(c["id"])) % (2 ** 31)
                out.append(c)

    # ---- forward, weight-stationary: BN 256 / 128 / 64, partial last column block, groups vs tiles_m edges
    f = "fwd_ws"
    add(f, "fwd", 300, 272, 256, bias="f32", relu=True)                    # BN 256, last block 16 wide, 1 tile / CTA
    add(f, "fwd", 1000, 272, 256, bias="16", addend=True, out="f32")       # fp32 out: two staging passes
    add(f, "fwd", 129, 320, 192, bias="16", addend=True)                   # last block 64 wide
    add(f, "fwd", 4099, 16, 512, bias="f32", relu=True, addend=True)       # BN 64, N = 16
    add(f, "fwd", 2000, 64, 1024, bias="16", out="f32")                    # BN 64 at the longest stationary reduction
    add(f, "fwd", 64 * sms, 256, 256, addend=True)                         # tiles_m == groups
    add(f, "fwd", 64 * sms + 1, 256, 256, bias="f32", relu=True, out="f32")   # tiles_m == groups + 1
    add(f, "fwd", 64 * (sms // 2) + 1, 512, 256, bias="16")                # two column blocks, tiles_m == groups + 1
    add(f, "fwd", 40000, 256, 256, addend=True)                            # encoder production shapes
    add(f, "fwd", 40000, 512, 256, bias="f32", relu=True)
    add(f, "fwd", 40000, 256, 512, bias="f32", addend=True)
    add(f, "fwd", 40000, 512, 512, bias="16")
    add(f, "fwd", 44511, 768, 256, bias="f32", out="f32")
    add(f, "fwd", 184950, 256, 256, bias="f32")
    add(f, "fwd", 1000, 192, 512, bias="f32", out="f32")
    add(f, "fwd", 1000, 256, 256, regimes=("exact",), bias="f32", special="ties")
    add(f, "fwd", 300, 256, 256, regimes=("exact",), dtypes=(torch.float16,), bias="f32", special="inf")
    add(f, "fwd", 300, 256, 256, regimes=("exact",), dtypes=(torch.float16,), special="subnormal")
    # NaN / inf locality: a NaN in x[m, k] makes row m NaN; inf x 0 gives NaN; every other element stays exact
    add(f, "fwd", 1000, 256, 256, regimes=("exact",), bias="f32",
        poison=(("a", (7, 3), float("nan")), ("a", (700, 100), float("inf"))))

    # ---- input gradient, weight-stationary (W read MN-major)
    f = "dgrad_ws"
    add(f, "dgrad", 300, 256, 320, addend=True)                            # BN 256, last block loads one chunk
    add(f, "dgrad", 1000, 512, 256)                                        # BN 128, ragged M
    add(f, "dgrad", 4099, 768, 64, addend=True)                            # BN 64
    add(f, "dgrad", 129, 1024, 128, addend=True)                           # BN 64 at the longest reduction
    add(f, "dgrad", 40000, 256, 256)
    add(f, "dgrad", 40000, 512, 256, addend=True)
    add(f, "dgrad", 40000, 256, 512)
    add(f, "dgrad", 40000, 768, 256)
    add(f, "dgrad", 184950, 256, 256, addend=True)
    add(f, "dgrad", 1000, 256, 256, regimes=("exact",), addend=True, special="ties")
    add(f, "dgrad", 1000, 256, 256, regimes=("exact",), poison=(("a", (5, 9), float("nan")),))

    # ---- streamed forward (reduction > 1024): BN 128 for N > 64, else 64
    f = "fwd_stream"
    add(f, "fwd", 300, 272, 1088, bias="f32", relu=True)
    add(f, "fwd", 1000, 64, 2048, bias="16", addend=True, out="f32")
    add(f, "fwd", 129, 48, 1088, bias="f32", relu=True, addend=True)
    add(f, "fwd", 513, 384, 2048, addend=True, out="f32")
    add(f, "fwd", 300, 272, 1088, regimes=("exact",), bias="f32", special="ties")
    add(f, "fwd", 300, 128, 1088, regimes=("exact",), dtypes=(torch.float16,), bias="f32", special="inf")
    add(f, "fwd", 300, 128, 1088, regimes=("exact",), dtypes=(torch.float16,), special="subnormal")
    add(f, "fwd", 300, 128, 1088, regimes=("exact",),
        poison=(("a", (131, 1000), float("nan")), ("a", (7, 2), float("inf"))))

    # ---- streamed input gradient (reduction N > 1024): BN 128 when K % 128 == 0, else 64
    f = "dgrad_stream"
    add(f, "dgrad", 300, 1152, 256, addend=True)
    add(f, "dgrad", 1000, 1152, 320, addend=True)
    add(f, "dgrad", 129, 2048, 128)
    add(f, "dgrad", 4099, 1088, 192, addend=True)

    # ---- weight gradient, fp32 reduction into dW (and db)
    f = "wgrad"
    s0 = -(-sms // 4)                                                      # splits of N = K = 256
    add(f, "wgrad", 1, 8, 64, db=True)                                     # one row, one split
    add(f, "wgrad", 63, 72, 320, db=True)                                  # one split, K % 128 != 0
    add(f, "wgrad", 65, 200, 256)                                          # two splits, the last of one row
    add(f, "wgrad", s0 * 192, 256, 256, db=True)                           # splits x rows == M exactly
    add(f, "wgrad", 10000, 768, 192, db=True)                              # many splits, short last split
    add(f, "wgrad", 4099, 8, 1088, db=True)
    add(f, "wgrad", 40000, 256, 256, db=True)
    add(f, "wgrad", 40000, 512, 256, db=True)
    add(f, "wgrad", 44511, 768, 256, db=True)
    add(f, "wgrad", 1000, 192, 512, db=True)
    add(f, "wgrad", 184950, 256, 256, db=True)
    add(f, "wgrad", 1000, 72, 256, regimes=("exact",), db=True, poison=(("a", (17, 40), float("nan")),))

    # ---- two-pass weight gradient: per-split slabs, then wgrad_reduce_kernel in the parameter's dtype
    f = "two_pass"
    for gdt in (torch.float32, torch.bfloat16, torch.float16):
        add(f, "wgrad_out", 65, 200, 256, db=True, grad_dtype=gdt)
        add(f, "wgrad_out", 10000, 768, 192, db=True, grad_dtype=gdt)
    add(f, "wgrad_out", 1, 8, 64, db=True, grad_dtype=torch.float32)
    add(f, "wgrad_out", 10000, 72, 320, grad_dtype=torch.float16)
    add(f, "wgrad_out", 184950, 256, 256, db=True, grad_dtype=torch.bfloat16)
    add(f, "wgrad_out", 1000, 72, 256, regimes=("exact",), db=True, grad_dtype=torch.bfloat16,
        poison=(("a", (17, 40), float("nan")),))
    add(f, "wgrad_into", 4099, 72, 320, db=True)
    add(f, "wgrad_into", 40000, 512, 256, db=True)

    # ---- an output whose flat index passes 2^31 elements (size_t epilogue offsets of the streamed kernel); only the
    # row blocks on both sides of the boundary are compared
    add("big", "fwd", (1 << 31) // 2048 + 256, 2048, 1088, regimes=("exact",), dtypes=(torch.bfloat16,), out="f32",
        cpu_gen=False, rows=((1 << 31) // 2048 - 256, (1 << 31) // 2048 + 256))
    return out
