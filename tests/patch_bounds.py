"""Per-element error bounds of the PATCHED packed Linear as the layer runs it (GGMLOps.Linear.forward_ggml_cast_weights with
LoRA, LoHa, LoKr or DoRA entries), the float64 restatement of comfy.lora.calculate_weight they are taken against, and the case
list of the layer's routes.

No GPU here: tests/test_patch_bounds.py checks these helpers on the CPU (restatement, coverage, mutations the bounds reject),
tests/test_gpu_patch_bounds.py applies them to the layer's output, element by element.

The restatement (`calculate_weight`, `ideal_weight`).  ComfyUI's arithmetic for the entries the layer serves, per entry in list
order: narrow W to the entry's offset (dim, start, size), multiply that by strength_model when it is not 1, form the delta in
the intermediate dtype (LoRA up @ down with a = alpha / rank, LoHa (w1a @ w1b) * (w2a @ w2b) with a = alpha / w1b.rows, LoKr
kron(w1, w2) with a decomposed factor the mm of its halves and a = alpha / that factor's rank, a = 1 for alpha None), then
either W += ((strength a) delta).to(W.dtype) or weight_decompose (DoRA; s = dora_scale / (norm + eps) over the rows of W
BEFORE the patch for dora_scale.shape[0] == rows, else over the columns of W + a delta).  `calculate_weight` runs that in W's
dtype on W's device (the reference's W_ref and its DoRA factors s); `ideal_weight` runs it in float64 without any rounding,
with the s of the act-dtype replay (as the reference computes them) -- W*.

The bounds.  Every route evaluates y = x W*^T + b through a factorisation of W*; each bound is the chain bound of
tests/linear_bounds.py on the factors the route multiplies, plus, for every rounding the route performs, the rounding's size
against the magnitude of what it rounds (never a blanket u_act |x| |W*|: that would hide a dropped row in bf16).  Notation:
u = 2^-23 (fp32, charged as linear_bounds does), u_a / eta_a the unit roundoff and half the smallest subnormal of the
activation dtype (fp16 2^-11 / 2^-25, bf16 2^-8 / 2^-134), u_h / eta_h those of fp16.  An operand is a pair (value, error
bound) in float64; the propagation rules are

  product   X W^T of (x, ex), (w, ew) by an fp32 chain over n terms:  |x| ew^T + ex |w|^T + ex ew^T + c n u (|x| + ex)(|w| + ew)^T
            (c = 2, n = inner size + 2; linear_bounds' derivation);
  rounding  of (v, e) to a dtype:  e + u_d (|v| + e) + eta_d.

In-kernel LoRA / LoHa (FUSED_TMEM + k-blocks, `kernel_bound`).  T* = x_band down^T (float64, exact), the layer's T = act(fl(x
act(down)^T)): error (u_a |down| + eta_a) through the product, the chain, then one rounding.  U* = scale up on the term's rows
(zero elsewhere), the layer's U = fp16(fp32(scale) fp32(up)) read by the MMA in the activation dtype: 2u relative, then the
fp16 rounding (relative u_h plus eta_h for fp16 subnormals), then for bf16 the bf16 rounding.  The kernel then forms
fl([x | T] [W0 | U]^T) + b over K' = K + 64 J: the product rule on those extended operands, the bias in the chain, u |v| for the
last add; the final rounding to the activation dtype is `linear_bounds.check`'s interval.  For LoHa the test's factorisation
is its own Khatri-Rao product (`khatri_rao`).

Side GEMMs (`side_bound`: `_add_lora`, band-wise or concatenated, and `lora_side_sum` under autograd).  The base route's bound
on W0, rounded to the activation dtype (y_base); per group of terms (one group per term when any term has a band, else one
concatenated group) t = act(fl(x_band act(down)^T)) as above, u = act(fp32(scale up)) (2u, then one act rounding), then the
addmm  y_band = act(fl(y_band + t u^T)): the product rule over r + 1 terms with y_band's own error carried, then one rounding.
Under autograd the product t u^T is rounded on its own before the add (one more rounding).

LoKr (`dequant_kron` + GEMM) and the two-step route.  The layer's weight IS the restated W_ref (checked bit for bit); the
output bound is the sharp linear bound of x W_ref^T + b (`linear_bounds.reference`); separately `weight_bound` bounds
|W_ref - W*| per element: per entry, the fp32 delta (c n u |factors| with n the rank, or u |kron| for whole LoKr factors,
then the scale's product u), the cast to W's dtype and the add, each rounding against its own magnitude; under
patch_dtype = "target" the delta's factors and products round in the activation dtype instead.

DoRA (`dora_kernel_bound`, `dora_side_bound`).  With the compact form W* = diag(r) W0 diag(c) + sum_j diag(rho_j) (a_j st_j
up_j down_j) diag(gamma_j) restated from the s factors (`dora_pieces`): in-kernel, xs = act(fp32(x) fp32(c)) (2u |x c|, one
rounding), T = act(fl(x act(down diag(gamma))^T)), U_j = act(fp16(fp32(a st rho up / r))) (u, then fp16, then act), acc =
fl([xs | T] [W0 | U]^T), y = fl(fp32(r) acc) + b: |r| times the product rule, u |r| |acc| for fp32(r), u |v| for the product and
u |v| for the bias add.  Side form: y_base = act(fl(fp32(r) fl(xs W0^T)) + b) as above without T, then t = act(fl(x act(down
diag gamma)^T)), up = act(a st rho up) (one rounding) and one addmm.

Non-finite entries (`reference_classes`): the layer's NaN / +Inf / -Inf pattern must be that of x W_ref^T + b with the
reference's own weight, `linear_bounds.classes`; a factorised evaluation sums the rank terms before an infinity meets them and
so cannot give that pattern (an Inf in `up` gives NaN in the reference, +-Inf from t u^T), so patch sets with non-finite factors
must take the two-step route.  Non-finite activations are a different contract: [x | T] [W0 | U]^T and x W'^T legitimately
differ there (a NaN in x reaches T and from there every feature a term covers, an Inf may become NaN or keep its sign), and
only "a non-finite x row gives a non-finite output row" is asserted (`nonfinite_activation_rows`).

How much of a bound is used.  `linear_bounds.check` reports the excess of |y - v| over half an output ulp, as a fraction of
the bound.  On the routes whose weight is the reference's own (LoKr, the two-step route) the only error left is the fp32
chain, which almost never exceeds half an ulp: fractions near 1e-4 are expected there, while a swapped LoKr band uses the
bound thousands of times over (tests/test_patch_bounds.py, tests/test_gpu_patch_bounds.py)."""
from dataclasses import dataclass, field

import torch

import linear_bounds as lb

U = lb.U
C = lb.C_BOUND
U_ACT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -24}
ETA = {torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -134, torch.float32: 2.0 ** -150}
ACT_CODE = {torch.float16: lb.F16, torch.bfloat16: lb.BF16}
_ADAPTERS = {"LoRAAdapter": "lora", "LoHaAdapter": "loha", "LoKrAdapter": "lokr"}


# ---------------------------------------------------------------- the restatement of calculate_weight
def parse(entry):
    """(strength, kind, payload, strength_model, offset) of a patch entry; the value is (kind, payload) or an adapter object."""
    value = entry[1]
    kind = _ADAPTERS.get(type(value).__name__)
    payload = tuple(value.weights) if kind is not None else tuple(value[1])
    kind = kind or value[0]
    return float(entry[0]), kind, payload, (entry[2] if len(entry) > 2 else 1.0), (entry[3] if len(entry) > 3 else None)


def delta(kind, p, dtype, device):
    """(delta, a, dora_scale): the entry's delta as calculate_weight forms it in `dtype`, alpha / rank, the DoRA tensor."""
    def c(t):
        return t.to(device=device, dtype=dtype)
    if kind == "lora":
        up, down, alpha = p[:3]
        a = 1.0 if alpha is None else float(alpha) / down.shape[0]
        return torch.mm(c(up).flatten(start_dim=1), c(down).flatten(start_dim=1)), a, (p[4] if len(p) > 4 else None)
    if kind == "loha":
        w1a, w1b, alpha, w2a, w2b = p[:5]
        a = 1.0 if alpha is None else float(alpha) / w1b.shape[0]
        return torch.mm(c(w1a), c(w1b)) * torch.mm(c(w2a), c(w2b)), a, (p[7] if len(p) > 7 else None)
    w1, w2, alpha, w1_a, w1_b, w2_a, w2_b = p[:7]
    dim = None
    if w1 is None:
        dim, w1 = w1_b.shape[0], torch.mm(c(w1_a), c(w1_b))
    if w2 is None:
        dim, w2 = w2_b.shape[0], torch.mm(c(w2_a), c(w2_b))
    a = float(alpha) / dim if alpha is not None and dim is not None else 1.0
    return torch.kron(c(w1), c(w2)), a, (p[8] if len(p) > 8 else None)


def _out_axis(dora_scale, W):
    return dora_scale.shape[0] == W.shape[0]


def weight_decompose(dora_scale, W, d, a, strength, intermediate):
    """ComfyUI's weight_decompose on a 2-D W, in place; returns the factor s (W's dtype, flat)."""
    ds = dora_scale.to(device=W.device, dtype=intermediate)
    d = d * a
    Wc = W + d.type(W.dtype)
    if _out_axis(dora_scale, W):
        nrm = W.reshape(W.shape[0], -1).norm(dim=1, keepdim=True).reshape(W.shape[0], 1)
    else:
        nrm = Wc.transpose(0, 1).reshape(W.shape[1], -1).norm(dim=1, keepdim=True).reshape(W.shape[1], 1).transpose(0, 1)
    nrm = nrm + torch.finfo(W.dtype).eps
    s = (ds.reshape(nrm.shape) / nrm).type(W.dtype)
    Wc *= s
    if strength != 1.0:
        Wc -= W
        W += strength * Wc
    else:
        W[:] = Wc
    return s.reshape(-1)


def calculate_weight(W, entries, intermediate=torch.float32):
    """The reference's patched weight, in place on W (its dtype and device): returns (W, [DoRA factor s or None per entry])."""
    factors = []
    for entry in entries:
        st, kind, p, sm, offset = parse(entry)
        Wb = W.narrow(*offset) if offset is not None else W
        if sm != 1.0:
            Wb *= sm
        d, a, ds = delta(kind, p, intermediate, W.device)
        d = d.reshape(Wb.shape)
        if ds is None:
            Wb += ((st * a) * d).type(Wb.dtype)
            factors.append(None)
        else:
            factors.append(weight_decompose(ds, Wb, d, a, st, intermediate))
    return W, factors


def ideal_weight(W0, entries, factors):
    """W*: the same patches in float64, never rounded, with the DoRA factors s of the act-dtype replay."""
    W = W0.to(torch.float64).clone()
    for entry, s in zip(entries, factors):
        st, kind, p, sm, offset = parse(entry)
        Wb = W.narrow(*offset) if offset is not None else W
        if sm != 1.0:
            Wb *= sm
        d, a, ds = delta(kind, p, torch.float64, W.device)
        d = a * d.reshape(Wb.shape)
        if s is None:
            Wb += st * d
            continue
        s = s.to(torch.float64)
        Wc = (Wb + d) * (s[:, None] if _out_axis(ds, Wb) else s[None, :])
        Wb += st * (Wc - Wb)
    return W


def reference_weights(W0, entries, intermediate=torch.float32):
    """(W_ref, W*, s factors) for the dequantised weight W0 (activation dtype)."""
    W_ref, factors = calculate_weight(W0.clone(), entries, intermediate)
    return W_ref, ideal_weight(W0, entries, factors), factors


# ---------------------------------------------------------------- the test's own factorisation
def khatri_rao(w1a, w1b, w2a, w2b):
    """LoHa (w1a w1b) * (w2a w2b) as one rank r1 r2 product up @ down, float64."""
    w1a, w1b, w2a, w2b = (t.to(torch.float64) for t in (w1a, w1b, w2a, w2b))
    up = torch.einsum("ni,nj->nij", w1a, w2a).reshape(w1a.shape[0], -1)
    down = torch.einsum("ik,jk->ijk", w1b, w2b).reshape(-1, w1b.shape[1])
    return up, down


@dataclass
class Term:
    """scale up @ down on a band (dim, start, size) or the whole weight; up / down float64 as the layer gets them (LoHa:
    `khatri_rao`), `down_src` the tensor the layer rounds to the activation dtype for T (LoRA: the entry's own down)."""
    scale: float
    up: torch.Tensor
    down: torch.Tensor
    band: tuple = None


def lora_terms(entries, device):
    """The LoRA-form terms of the LoRA / LoHa entries of a list (LoKr and DoRA entries skipped), in list order."""
    out = []
    for entry in entries:
        st, kind, p, _sm, offset = parse(entry)
        if kind == "lokr":
            continue
        if kind == "lora":
            up, down = (t.to(device=device, dtype=torch.float64) for t in p[:2])
            a = 1.0 if p[2] is None else float(p[2]) / down.shape[0]
        else:
            up, down = khatri_rao(*(t.to(device) for t in (p[0], p[1], p[3], p[4])))
            a = 1.0 if p[2] is None else float(p[2]) / p[1].shape[0]
        out.append(Term(st * a, up, down, None if offset is None else tuple(offset)))
    return out


def _extend(terms, N, K, M, x):
    """Per term: (rows slice, x columns used, T* [M, r], U* rows [size, r])."""
    out = []
    for t in terms:
        rows = slice(t.band[1], t.band[1] + t.band[2]) if t.band is not None and t.band[0] == 0 else slice(0, N)
        cols = slice(t.band[1], t.band[1] + t.band[2]) if t.band is not None and t.band[0] == 1 else slice(0, K)
        out.append((rows, cols))
    return out


# ---------------------------------------------------------------- propagation rules
def rnd(v, e, dtype):
    """Error bound after rounding a value v (known to within e) to `dtype`."""
    return e + U_ACT[dtype] * (v.abs() + e) + ETA[dtype]


def product(x, ex, w, ew, n=None):
    """Error bound of an fp32 chain x @ w^T with operand error bounds ex, ew (None = exact)."""
    n = (x.shape[1] if n is None else n) + 2
    ax, aw = x.abs(), w.abs()
    X = ax if ex is None else ax + ex
    W = aw if ew is None else aw + ew
    e = C * n * U * (X @ W.T)
    if ew is not None:
        e = e + ax @ ew.T
    if ex is not None:
        e = e + ex @ aw.T
        if ew is not None:
            e = e + ex @ ew.T
    return e


def _t_operand(x, cols, down, dt):
    """T = act(fl(x_band act(down)^T)): (T*, error bound)."""
    xs = x[:, cols]
    Tv = xs @ down.T
    return Tv, rnd(Tv, product(xs, None, down, U_ACT[dt] * down.abs() + ETA[dt], n=x.shape[1]), dt)


def _finite(t):
    return torch.where(torch.isfinite(t), t, torch.zeros_like(t))


def base_bound(x, W0, bias, ew0=None, mag=None):
    """(v, e) of the unpatched route's fp32 result x W0^T + b before its rounding: linear_bounds.reference, plus the weight
    operand's error bound ew0 (fast producers) and GEMV_FAST's sub-block magnitudes mag."""
    v, a, _cls = lb.reference(_finite(x), W0, bias, mag)
    if ew0 is not None:
        a = a + x.abs() @ ew0.T
    return v, a


def kernel_bound(x, W0, terms, dt, bias=None, ew0=None):
    """(v, a) of the in-kernel route y = act(fl([x | T] [W0 | U]^T) + b)."""
    M, K = x.shape
    N = W0.shape[0]
    R = sum(t.down.shape[0] for t in terms)
    Tv = torch.zeros(M, R, dtype=torch.float64, device=x.device)
    Te, Uv, Ue = torch.zeros_like(Tv), torch.zeros(N, R, dtype=torch.float64, device=x.device), None
    Ue = torch.zeros_like(Uv)
    r0 = 0
    for t, (rows, cols) in zip(terms, _extend(terms, N, K, M, x)):
        r = t.down.shape[0]
        Tv[:, r0:r0 + r], Te[:, r0:r0 + r] = _t_operand(x, cols, t.down, dt)
        u = t.scale * t.up
        eu = rnd(u, 2 * U * u.abs(), torch.float16)
        if dt == torch.bfloat16:
            eu = rnd(u, eu, dt)
        Uv[rows, r0:r0 + r], Ue[rows, r0:r0 + r] = u, eu
        r0 += r
    J = max(1, -(-R // 64))
    xh = torch.cat([x, Tv], 1)
    ex = torch.cat([torch.zeros_like(x), Te], 1)
    Wh = torch.cat([W0, Uv], 1)
    ew = torch.cat([torch.zeros_like(W0) if ew0 is None else ew0, Ue], 1)
    v = xh @ Wh.T
    a = product(xh, ex, Wh, ew, n=K + 64 * J)
    if bias is not None:
        v = v + bias[None, :]
        a = a + C * (K + 64 * J + 2) * U * bias.abs()[None, :]
    return v, a + U * v.abs()


def side_bound(x, W0, terms, dt, bias=None, ew0=None, mag=None, sidesum=False):
    """(v, a) of the side-GEMM route: the base route on W0, rounded, then `_add_lora` (or `lora_side_sum` when sidesum)."""
    M, K = x.shape
    N = W0.shape[0]
    v, a = base_bound(x, W0, bias, ew0, mag)
    a = rnd(v, a, dt)
    spans = _extend(terms, N, K, M, x)
    banded = sidesum or any(t.band is not None for t in terms)
    groups = [[i] for i in range(len(terms))] if banded else [list(range(len(terms)))]
    for g in groups:
        rows = spans[g[0]][0]
        T = [_t_operand(x, spans[i][1], terms[i].down, dt) for i in g]
        Tv, Te = torch.cat([t[0] for t in T], 1), torch.cat([t[1] for t in T], 1)
        u = torch.cat([terms[i].scale * terms[i].up for i in g], 1)
        eu = rnd(u, 2 * U * u.abs(), dt)
        d = Tv @ u.T
        ed = product(Tv, Te, u, eu)
        vb, ab = v[:, rows], a[:, rows]
        if sidesum:
            ed = rnd(d, ed, dt)
        new = vb + d
        e = ab + ed + C * (Tv.shape[1] + 3) * U * (vb.abs() + ab)
        v = v.clone()
        a = a.clone()
        v[:, rows] = new
        a[:, rows] = rnd(new, e, dt)
    return v, a


def weight_bound(W0, entries, W_star, intermediate=torch.float32, dt=None):
    """Per-element bound on |W_ref - W*| for entries without DoRA (LoKr, LoRA, LoHa), W0 in the activation dtype."""
    dt = W0.dtype if dt is None else dt
    W = W0.to(torch.float64).clone()
    e = torch.zeros_like(W)
    ui = U if intermediate == torch.float32 else U_ACT[intermediate]
    for entry in entries:
        st, kind, p, sm, offset = parse(entry)
        Wb = W.narrow(*offset) if offset is not None else W
        eb = e.narrow(*offset) if offset is not None else e
        if sm != 1.0:
            Wb *= sm
            eb.copy_(rnd(Wb, eb * abs(sm), dt))
        d, a, _ds = delta(kind, p, torch.float64, W.device)
        d = (st * a) * d.reshape(Wb.shape)
        if kind == "lora":
            mags = [(p[0], p[1])]
        elif kind == "loha":
            mags = [(p[0], p[1]), (p[3], p[4])]
        else:
            mags = [(p[3], p[4])] if p[0] is None else []
            mags += [(p[5], p[6])] if p[1] is None else []
        # each factor rounds to the intermediate dtype (not for fp32 factors), each mm is a chain, the products and the
        # kron / Hadamard product and the scale round once each: a relative bound (4 + chain) on |delta| of the magnitudes
        dm = abs(st * a) * delta(kind, tuple(t.abs() if torch.is_tensor(t) else t for t in p), torch.float64, W.device)[0].reshape(Wb.shape)
        n = max([f.shape[1] for f, _g in mags] or [1])
        ed = (C * (n + 2) * U + (10 * ui if intermediate != torch.float32 else 4 * U)) * dm
        ed = rnd(d, ed, dt)
        Wb += d
        eb.copy_(rnd(Wb, eb + ed, dt))
    return e


# ---------------------------------------------------------------- DoRA
@dataclass
class DoraPieces:
    """W* = diag(r) W0 diag(c) + sum_j diag(rho_j) (coef_j up_j down_j) diag(gamma_j), float64."""
    r: torch.Tensor
    c: torch.Tensor
    has_c: bool
    terms: list = field(default_factory=list)       # (coef, rho [N], gamma [K], up, down)


def dora_pieces(entries, factors, N, K, device):
    r = torch.ones(N, dtype=torch.float64, device=device)
    c = torch.ones(K, dtype=torch.float64, device=device)
    terms, has_c = [], False
    for entry, s in zip(entries, factors):
        st, kind, p, _sm, _offset = parse(entry)
        if kind == "lora":
            up, down = (t.to(device=device, dtype=torch.float64) for t in p[:2])
            a = 1.0 if p[2] is None else float(p[2]) / down.shape[0]
            ds = p[4] if len(p) > 4 else None
        else:
            up, down = khatri_rao(*(t.to(device) for t in (p[0], p[1], p[3], p[4])))
            a = 1.0 if p[2] is None else float(p[2]) / p[1].shape[0]
            ds = p[7] if len(p) > 7 else None
        ones_n, ones_k = torch.ones_like(r), torch.ones_like(c)
        if s is None:
            terms.append([st * a, ones_n, ones_k, up, down])
            continue
        s = s.to(device=device, dtype=torch.float64)
        f = 1.0 - st + st * s
        if ds.shape[0] == N:
            r = r * f
            for tm in terms:
                tm[1] = tm[1] * f
            terms.append([st * a, s, ones_k, up, down])
        else:
            c = c * f
            has_c = True
            for tm in terms:
                tm[2] = tm[2] * f
            terms.append([st * a, ones_n, s, up, down])
    return DoraPieces(r, c, has_c, [tuple(t) for t in terms])


def _dora_xs(x, pieces, dt):
    if not pieces.has_c:
        return x, None
    xs = x * pieces.c[None, :]
    return xs, rnd(xs, 2 * U * xs.abs(), dt)


def _dora_lowrank(x, pieces, dt):
    """T* = x down'^T with down' = down diag(gamma) (and the layer's error on T), and up' = coef diag(rho) up."""
    down = torch.cat([d * g[None, :] for _c, _rho, g, _u, d in pieces.terms], 0)
    up = torch.cat([coef * rho[:, None] * u for coef, rho, _g, u, _d in pieces.terms], 1)
    Tv = x @ down.T
    return Tv, rnd(Tv, product(x, None, down, U_ACT[dt] * down.abs() + ETA[dt]), dt), up


def dora_kernel_bound(x, W0, pieces, dt, bias=None, ew0=None):
    """(v, a) of ggufb200_linear_lora_scaled as the DoRA plan drives it."""
    K = x.shape[1]
    xs, exs = _dora_xs(x, pieces, dt)
    Tv, Te, up = _dora_lowrank(x, pieces, dt)
    r = pieces.r
    Uv = up / r[:, None]
    Ue = rnd(Uv, U * Uv.abs(), torch.float16)
    if dt == torch.bfloat16:
        Ue = rnd(Uv, Ue, dt)
    R = Tv.shape[1]
    J = max(1, -(-R // 64))
    xh, Wh = torch.cat([xs, Tv], 1), torch.cat([W0, Uv], 1)
    ex = torch.cat([torch.zeros_like(x) if exs is None else exs, Te], 1)
    ew = torch.cat([torch.zeros_like(W0) if ew0 is None else ew0, Ue], 1)
    acc = xh @ Wh.T
    eacc = product(xh, ex, Wh, ew, n=K + 64 * J)
    v = acc * r[None, :]
    a = eacc * r.abs()[None, :] + U * (r.abs()[None, :] * (acc.abs() + eacc)) + U * v.abs()
    if bias is not None:
        v = v + bias[None, :]
        a = a + U * bias.abs()[None, :]
    return v, a + U * v.abs()


def dora_side_bound(x, W0, pieces, dt, bias=None):
    """(v, a) of the DoRA side form: ggufb200_gemm_scaled on the dequantised weight, then one addmm."""
    K = x.shape[1]
    xs, exs = _dora_xs(x, pieces, dt)
    r = pieces.r
    acc = xs @ W0.T
    eacc = product(xs, exs, W0, None)
    v = acc * r[None, :]
    a = eacc * r.abs()[None, :] + U * (r.abs()[None, :] * (acc.abs() + eacc)) + U * v.abs()
    if bias is not None:
        v = v + bias[None, :]
        a = a + U * (v.abs() + bias.abs()[None, :])
    a = rnd(v, a, dt)
    Tv, Te, up = _dora_lowrank(x, pieces, dt)
    eu = rnd(up, torch.zeros_like(up), dt)
    d = Tv @ up.T
    e = a + product(Tv, Te, up, eu) + C * (Tv.shape[1] + 3) * U * (v.abs() + a)
    v = v + d
    return v, rnd(v, e, dt)


# ---------------------------------------------------------------- non-finite values
def reference_classes(x, W_ref, bias=None):
    """The reference's NaN / +Inf / -Inf pattern: x W_ref^T + b with its own patched weight."""
    return lb.classes(x, W_ref.to(torch.float64), bias)


def nonfinite_activation_rows(y, x):
    """The contract for non-finite activations: every token row with a NaN / Inf input is non-finite somewhere, every
    other row's class is untouched by it (checked by the caller on the finite rows)."""
    bad = ~torch.isfinite(x).all(1)
    return bool((~torch.isfinite(y[bad]).all(1)).all())


# ---------------------------------------------------------------- the case list
ROUTES = (
    "kernel",                # plain / banded LoRA in the FUSED_TMEM k-blocks, canonical weight
    "kernel_spans",          # ... reading the span-major copy (Q6_K)
    "kernel_straddled",      # ... on a straddled Q4_K weight (640 x 320)
    "side_gemv",             # side GEMMs on the M <= 8 GEMV (exact: GEMV, fast: GEMV_FAST)
    "side_rank513",          # total rank above the k-blocks' 512
    "side_no_kernel",        # lora_in_kernel = False
    "side_bf16_weight",      # a BF16 weight
    "side_dequant_dtype",    # dequant_dtype fp32
    "side_straddled_q6k",    # straddled Q6_K (no span copy for straddled weights)
    "side_fallback_sync",    # IQ2_XS on FUSED_SYNC
    "side_fallback_k1",      # TQ2_0 by K1 + GEMM
    "loha_kernel",
    "loha_side",
    "lokr",                  # LoKr alone: dequant_kron + GEMM
    "lokr_banded",
    "lokr_mixed",            # LoKr + LoRA + LoHa: kron + side GEMMs
    "lokr_two_step",         # 9 LoKr patches: more than dequant_kron applies
    "dora_kernel",
    "dora_side",
    "two_step",              # lora_side_gemm = False / patch_dtype "target" / strength_model != 1
    "autograd",              # lora_side_sum
    "nonfinite",             # non-finite factor entries: the reference's NaN / Inf pattern
)


@dataclass(frozen=True)
class PatchCase:
    """One forward of the patched layer.  `spec` names the patch list (tests/test_gpu_patch_bounds.py builds it)."""
    route: str
    spec: str
    qt: str = "Q4_K"
    N: int = 384
    K: int = 1024
    M: int = 33
    layer: tuple = ()        # (attribute, value) pairs set on the layer
    x3d: bool = False

    @property
    def id(self):
        extra = "".join(f"-{k}={v}" for k, v in self.layer)
        return f"{self.route}-{self.spec}-{self.qt}-{self.M}x{self.N}x{self.K}{extra}{'-3d' if self.x3d else ''}"


CASES = [
    # in-kernel LoRA: canonical, bands off the 8 / 64 / 128 grids, a partial last tile, J = 1, 2, 5, 8, ranks not multiples of 64
    PatchCase("kernel", "whole_r16", M=1),
    PatchCase("kernel", "whole_r16", M=9, x3d=True),
    PatchCase("kernel", "bands_offgrid", N=520, M=300),
    PatchCase("kernel", "bands_overlap", N=520, M=8),
    PatchCase("kernel", "cols_non64", M=33),
    PatchCase("kernel", "rank_J2", M=129),
    PatchCase("kernel", "rank_J5", M=300),
    PatchCase("kernel", "rank_J8", M=65),
    PatchCase("kernel", "strength_zero_neg", M=33),
    PatchCase("kernel", "u_subnormal", M=33),
    PatchCase("kernel", "slices_flux", N=2688, K=1024, M=64),
    PatchCase("kernel_spans", "bands_offgrid", qt="Q6_K", N=520, M=33),
    PatchCase("kernel_straddled", "bands_offgrid", N=640, K=320, M=129),
    PatchCase("side_gemv", "bands_offgrid", N=520, M=1, layer=(("lora_in_kernel", False),)),
    PatchCase("side_gemv", "whole_r16", M=8, layer=(("lora_in_kernel", False),)),
    PatchCase("side_rank513", "rank_513", M=33),
    PatchCase("side_no_kernel", "bands_offgrid", N=520, M=300, layer=(("lora_in_kernel", False),)),
    PatchCase("side_no_kernel", "whole_two", M=33, layer=(("lora_in_kernel", False),)),
    PatchCase("side_bf16_weight", "bands_offgrid", qt="BF16", N=520, M=33),
    PatchCase("side_dequant_dtype", "bands_offgrid", N=520, M=33, layer=(("dequant_dtype", torch.float32),)),
    PatchCase("side_straddled_q6k", "bands_offgrid", qt="Q6_K", N=640, K=320, M=33),
    PatchCase("side_fallback_sync", "bands_offgrid", qt="IQ2_XS", N=520, M=300),
    PatchCase("side_fallback_k1", "whole_r16", qt="TQ2_0", M=5),
    PatchCase("kernel", "u_above_f16", M=33),
    PatchCase("loha_kernel", "loha_4", M=33),
    PatchCase("loha_kernel", "loha_16", M=300),
    PatchCase("loha_side", "loha_32", M=33),
    PatchCase("lokr", "lokr_whole", M=33),
    PatchCase("lokr_banded", "lokr_bands", N=520, M=9),
    PatchCase("lokr_mixed", "lokr_mixed", N=768, M=33),
    PatchCase("lokr_two_step", "lokr_nine", M=33),
    PatchCase("dora_kernel", "dora_out", M=33),
    PatchCase("dora_kernel", "dora_in", M=300),
    PatchCase("dora_kernel", "dora_both", M=9),
    PatchCase("dora_side", "dora_both_r0", M=33),
    PatchCase("two_step", "mixed_whole", M=33, layer=(("lora_side_gemm", False),)),
    PatchCase("two_step", "mixed_whole", M=33, layer=(("patch_dtype", "target"),)),
    PatchCase("two_step", "strength_model", M=33),
    PatchCase("autograd", "bands_offgrid", N=520, M=33),
    PatchCase("nonfinite", "nan_up_band", N=520, M=33),
    PatchCase("nonfinite", "inf_down_band", N=520, M=300),
    PatchCase("nonfinite", "inf_up_whole", M=33),
    PatchCase("nonfinite", "nan_lokr", N=520, M=33),
]
