"""ORACLE (test infrastructure, not product code): float64 restatement of what d3r_criterion (dust3r_b200/csrc/criterion_ops.cu)
computes, with an error bound for every quantity it returns.

The oracle reads exactly what the kernel reads -- the fp32 T = inv(camera_pose of view 1) the caller passes, the fp32 points,
masks and confidences, the flags, dist_clip and alpha -- widened to float64 exactly.  So a difference from the kernel is the
kernel's own fp32 arithmetic, and the bounds below cover it element by element.

Notation: u = 2^-24 (one fp32 rounding), gamma(n) = n u / (1 - n u), u64 = 2^-53.  The build uses IEEE division and sqrtf
(no fast math); FMA contraction only removes roundings.  Every bound is absolute, per element, derived from the operations
of load_pixel / norm3 / loss_kernel with one term per rounding step; none is fitted to observations.
  transform   g_k = T_k0 x + T_k1 y + T_k2 z + T_k3: a four-term dot product,  dg_k = gamma(4) (sum_j |T_kj x_j| + |T_k3|)
              (+ dT (|x|_1 + 1) when T itself is uncertain by dT per element: the golden check, where the reference inverted
              the pose itself)
  norms       |v| = sqrtf(v0^2 + v1^2 + v2^2) of a v known to dv: three non-negative products and two additions (gamma(3)
              relative), the square root halves that and rounds once (u): d|v| = |dv|_1 + gamma(3) (|v| + |dv|_1)
  a - b, a * b, a / b   of values known to da, db: the propagated error plus one rounding u (|result| + propagated error);
              a / s: (da + |a| ds / |s|) / (|s| - ds), infinite when ds >= |s|
  masks       valid & (|g| <= dist_clip): bit-exact, except pixels with ||g| - dist_clip| <= d|g|, reported as undecided
  norm. factors  nf = sum_valid |v| / count (0 for no valid pixel), floored at 1e-8.  The reference writes the divisor as
              count + 1e-8, but count is an integer tensor and the sum is the default fp32 dtype, so the 1e-8 is lost to
              rounding for any count >= 1.  The kernel sums the fp32 norms in fp64 (count 2 u64 relative) and rounds once to
              fp32 (u): dnf = sum_valid d|v| / count + 2 count u64 nf + u (nf + dnf); the floor is 1-Lipschitz, its fp32
              constant 1e-8f adds u 1e-8
  medians     the device takes the same order statistic (element (count - 1) // 2 of the non-NaN values) of its own fp32
              column values, each within its element bound of the float64 one.  Order statistics are 1-Lipschitz in the sup
              norm, so |median - median64| <= the largest element bound of that column: ties and rank swaps caused by the
              rounding need no special case.  The prediction-scale clip to [1e-3, 1e3] is 1-Lipschitz (its fp32 constants add
              u |clipped value|).
  loss        l = |p - g| as above; conf * l - alpha * log(conf): logf is within 1 ulp (2 u relative) and the two products
              and the difference round once each: dcl = c dl + 3 u c (l + dl) + 5 u alpha |log c|
  per view    fixed-order fp64 sums of the fp32 per-pixel values (count 2 u64 relative), one division by the count and one
              rounding to fp32; out[4] adds one more fp32 rounding.  With fp32_sums (the reference, which sums in fp32 in any
              order) a sum of n terms adds gamma(n) times the sum of their magnitudes.
The loss pass runs twice in the tests: with the float64 stage parameters, for the end-to-end bound of the results, and with
the device's own stage parameters (P given, bound 0), for a per-pixel bound that depends on nothing the medians chose."""
from __future__ import annotations

from dataclasses import dataclass
from types import SimpleNamespace
from typing import Optional

import torch

U = 2.0 ** -24
U64 = 2.0 ** -53
F64 = torch.float64
NORM, GT_SCALE, SHIFT, SCALE, CONF, CLIP = 1, 2, 4, 8, 16, 32
# the kernel's per-pair parameters: P[field * B + b], in the order of `enum Field` in criterion_ops.cu
FIELDS = ['nf_gt', 'nf_pr', 'shift_gt', 'shift_pr', 'centre_gt_x', 'centre_gt_y', 'centre_gt_z', 'centre_pr_x', 'centre_pr_y',
          'centre_pr_z', 'scale_gt', 'scale_pr']
K_FIELDS = len(FIELDS)


def gamma(n):
    return n * U / (1 - n * U)


@dataclass
class Inputs64:
    """What one d3r_criterion call reads, in float64: T (B,4,4), per view gt / pr (B,n,3), valid (B,n) bool, conf (B,n)."""
    T: torch.Tensor
    gt: tuple
    valid: tuple
    pr: tuple
    conf: Optional[tuple]
    flags: int
    clip: float = 0.0
    alpha: float = 0.0
    dT: float = 0.0             # per-element uncertainty of T
    fp32_sums: bool = False     # bound the reference's fp32 sums instead of the kernel's fp64 ones

    @property
    def B(self):
        return self.T.shape[0]


def inputs64(T, gt1, gt2, valid1, valid2, pr1, pr2, conf1=None, conf2=None, *, flags, clip=0.0, alpha=0.0, **kw):
    """Widen the kernel's inputs (any float dtype, (B,H,W,3) or (B,n,3)) to float64 exactly."""
    B = T.shape[0]
    pts = lambda t: t.detach().cpu().to(F64).reshape(B, -1, 3)
    per = lambda t: t.detach().cpu().reshape(B, -1)
    conf = (per(conf1).to(F64), per(conf2).to(F64)) if flags & CONF else None
    return Inputs64(T.detach().cpu().to(F64).reshape(B, 4, 4), (pts(gt1), pts(gt2)), (per(valid1) != 0, per(valid2) != 0),
                    (pts(pr1), pts(pr2)), conf, flags, float(clip), float(alpha), **kw)


# ----------------------------------------------------------------------------------- bounded arithmetic: (value, bound)
def _round(v, e):
    return v, e + U * (v.abs() + e)


def _sub(a, da, b, db):
    return _round(a - b, da + db)


def _mul(a, da, s, ds):
    return _round(a * s, da * s.abs() + a.abs() * ds + da * ds)


def _div(a, da, s, ds):
    v = a / s
    e = (da + a.abs() * ds / s.abs()) / (s.abs() - ds)
    e = torch.where(s.abs() > ds, e, torch.full_like(e, float('inf')))
    return _round(v, e)


def _norm(v, dv):
    n = v.norm(dim=-1)
    e = dv.sum(-1)
    return n, e + gamma(3) * (n + e)


def _masked_sum(x, m):
    return torch.where(m, x, torch.zeros_like(x)).sum(-1)


def order_statistic(cols, upper=False):
    """Per row, element (count - 1) // 2 (torch.nanmedian's lower median; count // 2 with upper) of the non-NaN values,
    NaN for a row without one."""
    s = torch.sort(cols, dim=-1).values          # NaN sorts last
    cnt = (~cols.isnan()).sum(-1)
    k = (cnt // 2 if upper else (cnt - 1) // 2).clamp(min=0)
    med = s.gather(-1, k[:, None])[:, 0]
    return torch.where(cnt > 0, med, torch.full_like(med, float('nan')))


def _median(cols, dcols, valid, upper=False):
    """Joint median over both views of one column, and its bound: the largest element bound of the column."""
    c = torch.cat([torch.where(m, x, torch.full_like(x, float('nan'))) for x, m in zip(cols, valid)], dim=1)
    d = torch.cat([torch.where(m & ~x.isnan(), e, torch.zeros_like(e)) for x, e, m in zip(cols, dcols, valid)], dim=1)
    return order_statistic(c, upper), d.amax(dim=1)


def _nf(norms, dnorms, valid, inp, floor=True):
    cnt = sum(m.sum(-1) for m in valid).to(F64)
    s = sum(_masked_sum(x, m) for x, m in zip(norms, valid))
    ds = sum(_masked_sum(e, m) for e, m in zip(dnorms, valid))
    c1 = cnt.clamp(min=1)
    nf = s / c1
    e = ds / c1 + 2 * cnt * U64 * nf.abs()
    if inp.fp32_sums:
        e = e + gamma(sum(x.shape[1] for x in norms)) * s.abs() / c1
    nf, e = _round(nf, e)
    if floor:
        nf = nf.clamp(min=1e-8)
        e = e + U * 1e-8
    return nf, e


# ------------------------------------------------------------------------------------------------------------ criterion
def transform(inp, decide=None):
    """Per view: g = T gt (B,n,3), its bound, the valid mask after dist_clip and the undecided pixels.  `decide` (per view,
    e.g. the device's masks) settles the undecided pixels."""
    R, t = inp.T[:, None, :3, :3], inp.T[:, None, :3, 3]
    out = []
    for v in range(2):
        x = inp.gt[v]
        g = (R @ x[..., None])[..., 0] + t
        dg = gamma(4) * ((R.abs() @ x.abs()[..., None])[..., 0] + t.abs())
        if inp.dT:
            dg = dg + inp.dT * (x.abs().sum(-1, keepdim=True) + 1)
        valid, und = inp.valid[v].clone(), torch.zeros_like(inp.valid[v])
        if inp.flags & CLIP:
            ng, dng = _norm(g, dg)
            und = valid & ((ng - inp.clip).abs() <= dng)
            valid = valid & (ng <= inp.clip)
            if decide is not None:
                valid = torch.where(und, decide[v].reshape(valid.shape) != 0, valid)
        out.append((g, dg, valid, und))
    return out


def criterion64(inp, reduction, P=None, decide=None, upper_median=False, scale_clip=True, nf_floor=True):
    """Every stage of d3r_criterion in float64, with bounds.  reduction: 0 mean, 1 sum, 2 none.  P: the device's stage
    parameters (kFields, B) to use instead of the float64 ones (their bound is then 0).  upper_median / scale_clip /
    nf_floor: deliberate mistakes for the resolution checks."""
    f, B = inp.flags, inp.B
    views = transform(inp, decide)
    valid = [x[2] for x in views]
    par = {}

    def stage(name, val, err):
        if P is not None:
            i = FIELDS.index(name)
            val = P[i:i + (3 if name.startswith('centre') else 1)].to(F64).T.reshape(val.shape)
            err = torch.zeros_like(val)
        par[name.replace('_x', '')] = (val, err)
        return val, err

    # normalisation factors (the kernel computes both whatever the flags)
    ng = [_norm(g, dg) for g, dg, _, _ in views]
    npr = [_norm(p, torch.zeros_like(p)) for p in inp.pr]
    nfg, dnfg = stage('nf_gt', *_nf([x[0] for x in ng], [x[1] for x in ng], valid, inp, nf_floor))
    nfp, dnfp = stage('nf_pr', *_nf([x[0] for x in npr], [x[1] for x in npr], valid, inp, nf_floor))
    G = [(g, dg) for g, dg, _, _ in views]
    Pr = [(p, torch.zeros_like(p)) for p in inp.pr]
    col = lambda t: t[:, None, None]
    if f & NORM:
        Pr = [_div(p, dp, col(nfp), col(dnfp)) for p, dp in Pr]
        if not f & GT_SCALE:
            G = [_div(g, dg, col(nfg), col(dnfg)) for g, dg in G]
    if f & SHIFT:
        for name, pts in (('shift_gt', G), ('shift_pr', Pr)):
            s, ds = stage(name, *_median([x[0][..., 2] for x in pts], [x[1][..., 2] for x in pts], valid, upper_median))
            for k, (x, dx) in enumerate(pts):
                z, dz = _sub(x[..., 2], dx[..., 2], s[:, None], ds[:, None])
                pts[k] = (torch.cat([x[..., :2], z[..., None]], -1), torch.cat([dx[..., :2], dz[..., None]], -1))
    if f & SCALE:
        sc = {}
        for which, pts in (('gt', G), ('pr', Pr)):
            c = [_median([x[0][..., k] for x in pts], [x[1][..., k] for x in pts], valid, upper_median) for k in range(3)]
            c, dc = stage(f'centre_{which}_x', torch.stack([m for m, _ in c], -1), torch.stack([e for _, e in c], -1))
            rad = [_norm(*_sub(x, dx, c[:, None], dc[:, None])) for x, dx in pts]
            sc[which] = stage(f'scale_{which}', *_median([r for r, _ in rad], [e for _, e in rad], valid, upper_median))
        (sg, dsg), (sp, dsp) = sc['gt'], sc['pr']
        if scale_clip:
            clipped = sp.clamp(1e-3, 1e3)
            dsp = dsp + U * (clipped != sp) * clipped.abs()
            sp = clipped
        par['scale_pr_clipped'] = (sp, dsp)
        if f & GT_SCALE:
            fac, dfac = _div(sg, dsg, sp, dsp)
            Pr = [_mul(p, dp, col(fac), col(dfac)) for p, dp in Pr]
        else:
            G = [_div(g, dg, col(sg), col(dsg)) for g, dg in G]
            Pr = [_div(p, dp, col(sp), col(dsp)) for p, dp in Pr]

    # loss pass
    res = SimpleNamespace(valid=valid, undecided=[x[3] for x in views], params=par, l=[], dl=[], cl=[], dcl=[],
                          count=[int(m.sum()) for m in valid])
    out, dout = [0.0] * 7, [0.0] * 7
    for v in range(2):
        l, dl = _norm(*_sub(Pr[v][0], Pr[v][1], G[v][0], G[v][1]))
        res.l.append(l), res.dl.append(dl)
        m, n = valid[v], res.count[v]
        S, dS = float(_masked_sum(l, m).sum()), float(_masked_sum(dl, m).sum())
        dS += 2 * n * U64 * abs(S) + (gamma(n) * abs(S) if inp.fp32_sums else 0.0)
        if f & CONF:
            c = inp.conf[v]
            lc = c.log()
            cl = c * l - inp.alpha * lc
            dcl = c * dl + 3 * U * c * (l + dl) + 5 * U * inp.alpha * lc.abs()
            CS, dCS = float(_masked_sum(cl, m).sum()), float(_masked_sum(dcl, m).sum())
            dCS += 2 * n * U64 * float(_masked_sum(cl.abs(), m).sum())
            if inp.fp32_sums:
                dCS += gamma(n) * float(_masked_sum(cl.abs(), m).sum())
            res.cl.append(cl), res.dcl.append(dcl)
        else:
            CS = dCS = 0.0
        if reduction == 1:
            out[v], dout[v] = S, dS
        elif n > 0:
            out[v], dout[v] = S / n, dS / n
        else:
            out[v] = float('nan') if reduction == 2 else 0.0
        out[2 + v], dout[2 + v] = (CS / n, dCS / n) if n > 0 else (0.0, 0.0)
    for k in range(4):
        dout[k] += U * (abs(out[k]) + dout[k])
    if f & CONF:
        out[4], dout[4] = out[2] + out[3], dout[2] + dout[3]
    elif reduction == 2:
        out[4] = float('nan')
    else:
        out[4], dout[4] = out[0] + out[1], dout[0] + dout[1]
    dout[4] += U * (abs(out[4]) + dout[4])
    out[5], out[6] = res.count
    res.out, res.dout = out, dout
    res.pix = [l[m] for l, m in zip(res.l, valid)]
    res.dpix = [dl[m] for dl, m in zip(res.dl, valid)]
    return res


def params_tensor(res, B):
    """The float64 stage parameters of a criterion64 result in the kernel's (kFields, B) layout (NaN where not computed)."""
    P = torch.full((K_FIELDS, B), float('nan'), dtype=F64)
    for name, (val, _) in res.params.items():
        if name.startswith('centre'):
            i = FIELDS.index(name + '_x')
            P[i:i + 3] = val.T
        elif name in FIELDS:
            P[FIELDS.index(name)] = val
    return P


def ratio(err, bound):
    """Largest err / bound over the finite elements (NaN-pattern mismatches are checked separately); 0 when empty."""
    err, bound = torch.as_tensor(err, dtype=F64), torch.as_tensor(bound, dtype=F64)
    ok = ~err.isnan()
    if not bool(ok.any()):
        return 0.0
    r = err[ok] / bound[ok]
    r = torch.where(err[ok] == 0, torch.zeros_like(r), r)
    return float(r.max())
