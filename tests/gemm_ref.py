"""fp64 restatement of what nero_linear, nero_chain and nero_wgrad (+ the weight-norm finish) promise.

Everything here is written from the ABI text (include/nero_b200.h, the docstrings of nero_b200/ops.py), never from the
kernels, and is built from the layer PARAMETERS (weight_v / weight_g / bias), never from `w_eff` or the operand images,
which are kernel output.  The functions take the same descriptors the entry points take: ops.PreparedLayer, ops.Mat and
the ops.chain_layer dicts.  Long inputs are processed by the callers in row chunks (CHUNK rows), so nothing here holds
more than a few hundred MB at once.

Error bounds.  S = |A| |W_op|^T in fp64, the scale test_gemm_gpu.py uses; eps = 2^-23 is one fp32 rounding of the
stored result.  REL is the split-bf16 product error per unit of S: x = hi + lo with hi = bf16(x) (|x - hi| <= 2^-8 |x|) and
lo = bf16(x - hi) (|x - hi - lo| <= 2^-16 |x|), and the kernels drop lo_a lo_w, so one product is off by at most
3 * 2^-16 |a||w| = 4.6e-5 |a||w| (DESIGN.md "Error budget" quotes the typical 2e-5 of long sums, where the per-term errors
average out; a contraction over a single row, such as the transposed NeRF density head, reaches 2.06e-5 of S on real
data).  REL = 5e-5 adds the fp32 accumulation of the sum on top of that worst case.  TINY = 256 * 2^-126 covers the fp32
subnormals the tensor cores and the .ftz epilogue math flush to zero (at most one per product of a 256-deep contraction).

  bias kinds   REL |oscale| Lip (S + |bias|) + 2e-9 |oscale| (softplus ex2/lg2 approximation) + eps |ref|
               Lip = 1 (none, ReLU, softplus), 1/4 (sigmoid), exp(min(x, p)) (expclamp) at the fp64 pre-activation x.
               Sigmoid and expclamp use fp32 expf (<= 2 ulp, CUDA C Programming Guide, Table "single-precision
               mathematical functions"); sigmoid adds the rounding of 1 + t and of the division.  Their relative
               rounding is therefore <= 2^-22 + 2^-23 + 2^-24 < 2^-21, and their last term is 2^-21 |ref| instead of eps.
  DACT kinds   REL |oscale| |s| S + 2^-21 |oscale| |acc| (dsoftplus100_fast: ex2.approx plus the rounding of its
               argument) + eps |addend| + eps |ref|
  tail         REL |oscale| S + eps |ref|
  tangent out2 100 |V| (|1 - s| REL S + 2^-21 |acc|) + eps |ref|
  all          + TINY
  wgrad        per gradient tensor over the rows the calls cover: ||got - ref||_F <= 3e-5 ||scale||_F, the criterion of
               test_gemm_gpu.test_wgrad.  The scale is what the finish step's error is proportional to: the weight-norm
               map is linear in dW_r with ||d(dg_r)|| <= ||d(dW_r)|| (Cauchy-Schwarz) and ||d(dv_r)|| <= |g_r| / ||v_r||
               ||d(dW_r)|| (a projection), so scale = dW for dg and g / ||v|| dW for dv (dW itself for a plain weight);
               a bias sum is scaled by sum |dY|.  Measuring dg against ||dg|| instead would charge the kernel for the
               cancellation in dW_r . v_r.  nero_wgrad splits the M rows of one call over P = 66 slices and each slice
               accumulates its L = ceil(M / P) products in fp32 in order; with independent roundings the accumulated
               error of one entry stays within 2^-24 sqrt(L) sum_m |dY_m X_m| (the probabilistic bound of sequential
               summation, Higham, "Accuracy and Stability of Numerical Algorithms", sec. 4.2).  Stage II reaches
               L ~ 1.2e4 (7.6e5 rows per light-MLP call), where this term exceeds 3e-5 ||dW||; the bound therefore adds
               ||2^-24 sqrt(L) |dY|^T |X|||_F, carried through the same maps (|g| / ||v|| for dv).

When a chain layer's input is not stored by the kernel (the previous layer has no `save`), the reference propagates its
own fp64 result through that layer; the previous layer's bound B then enters the next layer as the input scale
|A| + B / REL, so that REL S covers both the product error and the propagated input error (B |W|^T).
"""
import torch

CHUNK = 65536
EPS = 2.0 ** -23
REL = 5e-5
TINY = 256 * 2.0 ** -126

# epilogue kinds (ops.EK_*) and codes of include/nero_b200.h
EK_BIAS_SOFTPLUS, EK_BIAS_RELU, EK_BIAS_GENERIC, EK_DACT_SOFTPLUS, EK_DACT_RELU, EK_DACT_NONE, EK_TANGENT = range(7)
KIND_NAMES = ('BIAS_SOFTPLUS', 'BIAS_RELU', 'BIAS_GENERIC', 'DACT_SOFTPLUS', 'DACT_RELU', 'DACT_NONE', 'TANGENT')
ACT_NONE, ACT_SOFTPLUS100, ACT_RELU, ACT_SIGMOID, ACT_EXPCLAMP = range(5)
EPI_BIAS_ACT, EPI_MUL_DACT, EPI_TANGENT = range(3)
BIAS_KINDS = (EK_BIAS_SOFTPLUS, EK_BIAS_RELU, EK_BIAS_GENERIC)


def ceil_div(a, b):
    return (a + b - 1) // b


def linear_kind(mode, act, H, dact):
    """The EpiKind an nero_linear call selects (nero_b200.h 'mode BIAS_ACT / MUL_DACT / TANGENT'; MUL_DACT without H or
    with dact = 0 multiplies by nothing)."""
    if mode == EPI_BIAS_ACT:
        return {ACT_SOFTPLUS100: EK_BIAS_SOFTPLUS, ACT_RELU: EK_BIAS_RELU}.get(act, EK_BIAS_GENERIC)
    if mode == EPI_TANGENT:
        return EK_TANGENT
    if H is None or dact == ACT_NONE:
        return EK_DACT_NONE
    return EK_DACT_RELU if dact == ACT_RELU else EK_DACT_SOFTPLUS


def kind_act(kind, act):
    """Activation a bias kind applies (nero_chain_layer: 0 bias+softplus100, 1 bias+relu, 2 bias+act)."""
    return {EK_BIAS_SOFTPLUS: ACT_SOFTPLUS100, EK_BIAS_RELU: ACT_RELU}.get(kind, act)


# ------------------------------------------------------------------------------------------------ weights
def effective_rows(layer):
    """Rows [row0, row0 + nrows) of g v / ||v|| (norm over the full reference row), or of `weight` when g is None
    (nero_prep_weight: 'W = g * v/||v||', 'g == NULL: plain weight')."""
    v = layer.weight.detach().double()[layer.row0:layer.row0 + layer.nrows]
    if layer.g is None:
        return v
    g = layer.g.detach().double()[layer.row0:layer.row0 + layer.nrows].reshape(-1, 1)
    return g * v / v.norm(dim=1, keepdim=True)


def layout_weight(layer):
    """[nrows, k_layout] effective weights in layout columns: reference column j goes to layout column kmap[j]
    (PreparedLayer: 'kmap : reference input column -> layout column'); all other layout columns are zero."""
    W = effective_rows(layer)
    out = torch.zeros(layer.nrows, max(layer.k_layout, 1), dtype=torch.float64, device=W.device)
    cols = torch.arange(layer.K, device=W.device) if layer.kmap_host is None else torch.tensor(layer.kmap_host, device=W.device)
    out[:, cols] = W
    return out


def operand(layer, transposed):
    """(W_op [n_pad, 64 k_chunks], k_valid): out = A[:, :64 k_chunks] W_op^T.  Forward use contracts over layout columns;
    transposed use reads layout columns [t_c0, t_c0 + t_ncols) and contracts over the nrows outputs
    (PreparedLayer: 't_cols : (c0, ncols) layout columns for which input gradients are needed')."""
    Wl = layout_weight(layer)
    if transposed:
        c0, nc = layer.t_cols
        n_pad, kc, kv = layer.t_npad, layer.t_chunks, ceil_div(layer.nrows, 4) * 4
        core = Wl[:, c0:c0 + nc].t()                     # [t_ncols, nrows]
    else:
        n_pad, kc, kv = layer.n_pad, layer.k_chunks, layer.k_valid
        core = Wl                                        # [nrows, k_layout]
    W = torch.zeros(n_pad, 64 * kc, dtype=torch.float64, device=Wl.device)
    W[:core.shape[0], :core.shape[1]] = core
    return W, kv


# ------------------------------------------------------------------------------------------------ epilogues
def act_fp64(x, act, p):
    if act == ACT_SOFTPLUS100:
        return torch.nn.functional.softplus(x, beta=100)
    if act == ACT_RELU:
        return torch.relu(x)
    if act == ACT_SIGMOID:
        return torch.sigmoid(x)
    if act == ACT_EXPCLAMP:
        return torch.exp(torch.clamp(x, max=p))
    return x


def act_lip(x, act, p):
    if act == ACT_SIGMOID:
        return torch.full_like(x, 0.25)
    if act == ACT_EXPCLAMP:
        return torch.exp(torch.clamp(x, max=p))
    return torch.ones_like(x)


def dact_s(kind, h, hscale):
    """Derivative factor from the STORED activation h: H > 0 for ReLU, 1 - exp(-100 hscale h) for softplus
    (nero_linear: 'act'(H*hscale)'; common.cuh dsoftplus100_from_h)."""
    if kind == EK_DACT_RELU:
        return (h > 0).double()
    if kind in (EK_DACT_SOFTPLUS, EK_TANGENT):
        return -torch.expm1(-100.0 * hscale * h)
    return torch.ones_like(h)


def epilogue(kind, acc, S, d, ins):
    """Reference of one layer's outputs on one row chunk.

    acc, S : [m, n_pad] fp64 product and its scale |A| |W_op|^T
    d      : descriptor with ncol_out, ncol_main, oscale, act, act_param, hscale and `bias` (fp64 vector or None)
    ins    : fp64 operand windows 'H', 'V', 'addend' ([m, nmain] or None)
    Returns (nmain, {'main': (ref, bound), 'tail': (ref, bound), 'out2': (ref, bound)}) restricted to the columns each
    output covers: main [0, nmain), tail [ncol_main, ncol_out) (DACT kinds), out2 [0, nmain) (TANGENT)."""
    nco, osc = d['ncol_out'], float(d['oscale'])
    aosc = abs(osc)
    res = {}
    if kind in BIAS_KINDS:
        nmain = nco
        a, s_ = acc[:, :nmain], S[:, :nmain]
        b = torch.zeros(nmain, dtype=torch.float64, device=acc.device)
        if d['bias'] is not None:
            nb = min(nmain, d['bias'].numel())
            b[:nb] = d['bias'][:nb]                    # 'oscale * act(acc + bias[col < n_bias])'
        x = a + b
        act = kind_act(kind, d['act'])
        ref = osc * act_fp64(x, act, d['act_param'])
        rnd = 2.0 ** -21 if act in (ACT_SIGMOID, ACT_EXPCLAMP) else EPS
        bound = REL * aosc * act_lip(x, act, d['act_param']) * (s_ + b.abs()) + rnd * ref.abs()
        if act == ACT_SOFTPLUS100:
            bound = bound + 2e-9 * aosc
        res['main'] = (ref, bound + TINY)
        return nmain, res
    nmain = min(nco, d['ncol_main'])
    a, s_ = acc[:, :nmain], S[:, :nmain]
    s = dact_s(kind, ins['H'], d['hscale']) if kind != EK_DACT_NONE else torch.ones_like(a)
    ref = osc * s * a
    bound = REL * aosc * s.abs() * s_ + 2.0 ** -21 * aosc * a.abs()
    if ins.get('addend') is not None:                            # '(+ addend)'; a chain's TANGENT layer has none
        ref = ref + ins['addend']
        bound = bound + EPS * ins['addend'].abs()
    res['main'] = (ref, bound + EPS * ref.abs() + TINY)
    if kind == EK_TANGENT:                                       # 'out2 = 100 * (1 - act'(H*hscale)) * V * acc'
        V = ins['V']
        r2 = 100.0 * (1.0 - s) * V * a
        res['out2'] = (r2, 100.0 * V.abs() * ((1.0 - s).abs() * REL * s_ + 2.0 ** -21 * a.abs()) + EPS * r2.abs() + TINY)
    if nco > d['ncol_main']:                                     # 'tail[:, :] = oscale * acc[:, ncol_main:]'
        at, st = acc[:, d['ncol_main']:nco], S[:, d['ncol_main']:nco]
        rt = osc * at
        res['tail'] = (rt, REL * aosc * st + EPS * rt.abs() + TINY)
    return nmain, res


# ------------------------------------------------------------------------------------------------ weight gradients
def wgrad_layout(dY, n_valid, X, k_valid, dY2=None, X2=None):
    """dW_layout = dY[:, :n_valid]^T X[:, :k_valid] (+ dY2^T X2) and the bias sums of dY only (nero_wgrad:
    'partial += dY^T X (+ dY2^T X2)', 'the column sums of dY'), with |dY|^T |X| and sum |dY|, for one row chunk of fp32
    inputs."""
    a = dY[:, :n_valid].double()
    dW = a.t() @ X[:, :k_valid].double()
    if dY2 is not None:
        dW = dW + dY2[:, :n_valid].double().t() @ X2[:, :k_valid].double()
    dWa = a.abs().t() @ X[:, :k_valid].double().abs()
    if dY2 is not None:
        dWa = dWa + dY2[:, :n_valid].double().abs().t() @ X2[:, :k_valid].double().abs()
    return dW, dWa, a.sum(0), a.abs().sum(0)


def wgrad_finish(layer, dW_layout, dWa_layout, db, db_abs, acc_rel):
    """Undo kmap and apply the weight-norm chain rule (nero_wgrad_finish: 'reduce partials, undo kmap, weight-norm chain
    rule'): dg_r = dW_r . v_r / ||v_r||, dv_r = g_r / ||v_r|| (dW_r - dg_r v_r / ||v_r||).  Returns one
    (ref, scale, accumulation term) triple each for dv (or dW of a plain weight) [nrows, K], dg [nrows, 1] (None for a plain
    weight) and the bias [nrows], in fp64; acc_rel = 2^-24 sqrt(L) scales |dY|^T |X| and sum |dY| (module docstring)."""
    n, kv = dW_layout.shape
    dev = dW_layout.device
    cols = torch.arange(layer.K, device=dev) if layer.kmap_host is None else torch.tensor(layer.kmap_host, device=dev)

    def unmap(t):
        full = torch.zeros(layer.nrows, max(layer.k_layout, kv), dtype=torch.float64, device=dev)
        full[:n, :kv] = t
        return full[:, cols]
    dW, dWa = unmap(dW_layout), unmap(dWa_layout) * acc_rel
    bias, babs = (torch.zeros(layer.nrows, dtype=torch.float64, device=dev) for _ in range(2))
    bias[:db.numel()] = db
    babs[:db_abs.numel()] = db_abs
    fb = (bias, babs, babs * acc_rel)
    if layer.g is None:
        return (dW, dW, dWa), None, fb
    v = layer.weight.detach().double()[layer.row0:layer.row0 + layer.nrows]
    g = layer.g.detach().double()[layer.row0:layer.row0 + layer.nrows].reshape(-1, 1)
    nv = v.norm(dim=1, keepdim=True)
    dg = (dW * v).sum(1, keepdim=True) / nv
    dv = g / nv * (dW - dg * v / nv)
    return (dv, g / nv * dW, g.abs() / nv * dWa), (dg, dW, dWa), fb


def frob_ok(got, ref, scale, acc, rel=3e-5):
    e, r = float((got - ref).norm()), rel * float(scale.norm()) + float(acc.norm())
    return e <= r, e, r
