"""Float64 Net::Backward in torch, on whatever device its inputs are on: a restatement of OracleNet.backward (oracle/net.py) with
Caffe's need-backward pruning (tests/stack_oracle.py), fast enough to run the training graphs at their real shape.

It differentiates at given activations: `blobs` maps a blob name to its forward value (the engine's own blobs, as
test_flownet_c_backward_matches_oracle does), and the ReLU derivative is read from the ReLU's top data, as oracle.relu_bwd
does, so a pre-activation within rounding of zero cannot take different sides of the kink here and in the engine.  Loss tops
are seeded with their loss_weight; a blob read by several layers sums the contributions (SplitLayer::Backward); a layer needs
backward when it has a parameter with lr_mult != 0 or a bottom that carries a gradient, and its type allows backward; a
bottom receives a gradient only if it carries one and its propagate_down is not false; a layer whose parameters all have
lr_mult 0 reports no parameter gradient.

Backward exists for the layer types on the trained paths of the training graphs: Convolution and Deconvolution (torch's
float64 convolution and its adjoints, weights shared between several bottoms), ReLU with negative_slope, Concat, Eltwise SUM,
Correlation of FlowNet2-C's class (tests/corr_ref.py: one shifted multiply-add per displacement) and L1Loss.  The layers that
only run forward there (DataAugmentation, Downsample, FlowAugmentation, Resample, FlowWarp, ChannelNorm) must not need it.
`conv_forward` is the layer-local forward of a Convolution or Deconvolution, with the ReLUs that run in place on its tops.

tests/test_net_grad64_cpu.py pins every piece to the oracle.
"""
import torch
import torch.nn.functional as F

from oracle.net import OracleNet, _hw, get, getall, parse_prototxt
from tests import corr_ref
from tests.stack_oracle import NO_BACKWARD, lr_mults

f64 = torch.float64

CONV = ("Convolution", "Deconvolution")


def conv_geometry(l):
    """(deconv, (sh, sw), (ph, pw), bias_term) of a Convolution or Deconvolution layer."""
    cp = get(l, "convolution_param")
    return (get(l, "type") == "Deconvolution", _hw(cp, "stride", "stride_h", "stride_w", 1), _hw(cp, "pad", "pad_h", "pad_w", 0),
            get(cp, "bias_term", "true") == "true")


# ---- L1Loss (l1loss_layer.cu: FindNotNaNs, KillMasked, the per-location L2 norm, MaskPlateauValues) ------------------------
def _l1_parts(b0, b1, l2_per_location, l2_prescale_by_channels, normalize_by_num_entries, plateau):
    d = b0.to(f64) if b1 is None else b0.to(f64) - b1.to(f64)
    ok = d == d
    N, C = d.shape[0], d.shape[1]
    norm = ok.sum().to(f64) / C if normalize_by_num_entries else torch.tensor(float(N), dtype=f64, device=d.device)
    dz = torch.where(ok, d, torch.zeros((), dtype=f64, device=d.device))
    if l2_per_location:
        w = 1.0 / C if l2_prescale_by_channels else 1.0
        ssum = (w * dz * dz).sum(1)
        kill = ssum.abs() < plateau * plateau if plateau > 0 else torch.zeros_like(ssum, dtype=torch.bool)
        return d, ok, norm, dz, w, torch.where(kill, torch.zeros((), dtype=f64, device=d.device), ssum), kill
    keep = ok & ~(d.abs() < plateau) if plateau > 0 else ok
    return d, keep, norm, dz, None, None, None


def l1loss_fwd64(b0, b1=None, l2_per_location=False, l2_prescale_by_channels=False, normalize_by_num_entries=False,
                 epsilon=1e-2, plateau=0.0):
    """The loss as a float64 scalar tensor: sum over locations of sqrt(sum_c w d^2 + epsilon) (or of |d|), divided by N (or by
    the count of non-NaN entries over C)."""
    d, keep, norm, dz, w, ssum, kill = _l1_parts(b0, b1, l2_per_location, l2_prescale_by_channels, normalize_by_num_entries,
                                                 plateau)
    if l2_per_location:
        return torch.sqrt(ssum + epsilon).sum() / norm
    return torch.where(keep, d, torch.zeros((), dtype=f64, device=d.device)).abs().sum() / norm


def l1loss_bwd64(b0, b1=None, top_diff=1.0, l2_per_location=False, l2_prescale_by_channels=False, normalize_by_num_entries=False,
                 epsilon=1e-2, plateau=0.0):
    """-> (bottom 0 diff, bottom 1 diff) in float64.  A masked entry gets 0; an unmasked |d| loss entry with d <= 0 gets -1, as
    the reference's sign kernel gives."""
    d, keep, norm, dz, w, ssum, kill = _l1_parts(b0, b1, l2_per_location, l2_prescale_by_channels, normalize_by_num_entries,
                                                 plateau)
    alpha = float(top_diff) / norm
    zero = torch.zeros((), dtype=f64, device=d.device)
    if l2_per_location:
        gs = torch.where(kill, zero, 0.5 / torch.sqrt(ssum + epsilon)) * alpha
        g = torch.where(keep, 2 * dz * (w * gs)[:, None], zero)
    else:
        g = torch.where(keep, alpha * torch.where(dz > 0, 1.0, -1.0).to(f64), zero)
    return g, -g


# ---- the layers ------------------------------------------------------------------------------------------------------------
def conv_backward64(x, w, td, deconv, stride, pad, need_x=True):
    """-> (bottom diff or None, weight diff, bias diff) of one bottom of a Convolution / Deconvolution, all float64; weights in
    Caffe layout (conv [Co][Ci][kh][kw], deconv [Ci][Co][kh][kw])."""
    x, w, td = x.to(f64), w.to(f64), td.to(f64)
    if deconv:        # the deconvolution is the convolution with the roles of bottom and top exchanged
        gx = F.conv2d(td, w, None, stride, pad) if need_x else None
        gw = torch.nn.grad.conv2d_weight(td, w.shape, x, stride, pad)
    else:
        gx = torch.nn.grad.conv2d_input(x.shape, w, td, stride, pad) if need_x else None
        gw = torch.nn.grad.conv2d_weight(x, w.shape, td, stride, pad)
    return gx, gw, td.sum((0, 2, 3))


def relu_backward64(top, td, slope):
    t = top.to(f64)
    return td * ((t > 0).to(f64) + slope * (t <= 0).to(f64))


def correlation_backward64(l, b0, b1, td):
    cp = get(l, "correlation_param")
    pad, k, md = int(get(cp, "pad", 0)), int(get(cp, "kernel_size")), int(get(cp, "max_displacement"))
    s1, s2 = int(get(cp, "stride_1", 1)), int(get(cp, "stride_2", 1))
    if (get(cp, "correlation_type", "MULTIPLY"), k, s1, pad) != ("MULTIPLY", 1, 1, md) or md % s2:
        raise NotImplementedError("backward of a correlation outside FlowNet2-C's class: %s" % get(l, "name"))
    return corr_ref.gradients(b0, b1, td, md, s2)


class NetGrad64(object):
    """prototxt: the filled text of a net.  params: {layer name: [weight, bias]} tensors (any float type), converted to float64 on
    the device of the blobs they meet."""

    def __init__(self, prototxt, params):
        self.root = parse_prototxt(prototxt)
        self.layers = [l for l in getall(self.root, "layer") if get(l, "type") != "Input"]
        self.by_name = {get(l, "name"): l for l in self.layers}
        self.params = params
        inputs = getall(self.root, "input") + [t for l in getall(self.root, "layer") if get(l, "type") == "Input"
                                               for t in getall(l, "top")]
        blob_need = {n: get(self.root, "force_backward", "false") == "true" for n in inputs}
        self.layer_need = {}
        for l in self.layers:
            need = any(lr != 0 for lr in lr_mults(l)) or any(blob_need.get(b, False) for b in getall(l, "bottom"))
            need = need and get(l, "type") not in NO_BACKWARD
            self.layer_need[get(l, "name")] = need
            for t in getall(l, "top"):
                blob_need[t] = need or blob_need.get(t, False)
        self.blob_need = blob_need

    def trained(self):
        """Names of the layers that report parameter gradients."""
        return [get(l, "name") for l in self.layers if self.layer_need[get(l, "name")] and any(lr != 0 for lr in lr_mults(l))]

    def losses(self):
        return [get(l, "name") for l in self.layers if get(l, "type") == "L1Loss"]

    def _param(self, name, i, like):
        return torch.as_tensor(self.params[name][i]).to(device=like.device, dtype=f64)

    # ---- forward of single layers --------------------------------------------------------------------------------------------
    def conv_forward(self, name, blobs):
        """{top: value} of Convolution / Deconvolution `name` on its bottoms from `blobs`, in float64, followed by the ReLUs that
        run in place on its tops (what the top blobs hold after the forward)."""
        l = self.by_name[name]
        deconv, s, p, bias = conv_geometry(l)
        out = {}
        for b, t in zip(getall(l, "bottom"), getall(l, "top")):
            x = blobs[b].to(f64)
            w = self._param(name, 0, x)
            bb = self._param(name, 1, x).reshape(-1) if bias else None
            out[t] = (F.conv_transpose2d if deconv else F.conv2d)(x, w, bb, s, p)
        for r in self.layers[self.layers.index(l) + 1:]:
            bots, tops = getall(r, "bottom"), getall(r, "top")
            if get(r, "type") == "ReLU" and bots == tops and tops[0] in out:
                y = out[tops[0]]
                out[tops[0]] = torch.where(y > 0, y, y * float(get(get(r, "relu_param", []), "negative_slope", 0)))
        return out

    def loss(self, name, blobs):
        """The float64 value of L1Loss `name` on its bottoms from `blobs`."""
        l = self.by_name[name]
        bots = [blobs[b] for b in getall(l, "bottom")]
        return l1loss_fwd64(bots[0], bots[1] if len(bots) > 1 else None, **OracleNet._l1_args(l))

    # ---- backward ----------------------------------------------------------------------------------------------------------------
    def backward(self, blobs, seeds=None, keep=None):
        """Net::Backward over the activations `blobs` (a mapping name -> tensor, read only where a layer needs the values; it
        may offer shape_of(name) for the concat bottoms, whose shapes alone are needed).
        seeds: {blob: top diff} besides the loss_weight seeds of the loss tops.  keep: names of the blob diffs to return (None:
        every one); the others are dropped once their producer has consumed them.  -> ({blob: diff}, {layer: [param diffs]})."""
        D = {k: torch.as_tensor(v).to(f64) for k, v in (seeds or {}).items()}
        for l in self.layers:
            if get(l, "type").endswith("Loss"):
                t = getall(l, "top")[0]
                if t not in D:
                    lw = getall(l, "loss_weight")
                    D[t] = torch.full((1,), float(lw[0]) if lw else 1.0, dtype=f64)
        P = {}
        for l in reversed(self.layers):
            name, typ = get(l, "name"), get(l, "type")
            tops, bots = getall(l, "top"), getall(l, "bottom")
            if not any(t in D for t in tops) or not self.layer_need[name]:
                continue
            if typ in NO_BACKWARD:
                continue
            pd = getall(l, "propagate_down")
            want = [self.blob_need.get(b, False) and not (i < len(pd) and pd[i] == "false") for i, b in enumerate(bots)]
            tds = [D.get(t) for t in tops]
            grads = self._backward_layer(l, blobs, bots, tops, tds, want, P)
            for t in tops:
                if t not in bots and keep is not None and t not in keep:
                    D.pop(t, None)
            for b, g, wnt in zip(bots, grads, want):
                if g is None or not wnt:
                    continue
                D[b] = g if (b in tops or b not in D) else D[b] + g
        return D, P

    def _backward_layer(self, l, blobs, bots, tops, tds, want, P):
        typ, name = get(l, "type"), get(l, "name")
        if typ in CONV:
            deconv, s, p, bias = conv_geometry(l)
            out, dw, db = [], 0, 0
            for b, td, wnt in zip(bots, tds, want):
                if td is None:
                    out.append(None)
                    continue
                x = blobs[b]
                td = td.to(x.device)
                gx, gw, gb = conv_backward64(x, self._param(name, 0, x), td, deconv, s, p, need_x=wnt)
                out.append(gx)
                dw, db = dw + gw, db + gb
            lrs = lr_mults(l)
            if any(lr != 0 for lr in lrs):
                P[name] = [dw] + ([db] if bias else [])
            return out
        if any(td is None for td in tds):
            raise NotImplementedError("%s %s: a top without a diff" % (typ, name))
        if typ == "ReLU":
            return [relu_backward64(blobs[tops[0]], tds[0].to(f64), float(get(get(l, "relu_param", []), "negative_slope", 0)))]
        if typ == "Eltwise":
            ep = get(l, "eltwise_param", [])
            if get(ep, "operation", "SUM") != "SUM":
                raise NotImplementedError("Eltwise %s" % get(ep, "operation"))
            coeffs = [float(c) for c in getall(ep, "coeff")] or [1.0] * len(bots)
            return [c * tds[0] for c in coeffs]
        if typ == "Concat":
            out, c0 = [], 0
            shape_of = getattr(blobs, "shape_of", lambda b: blobs[b].shape)
            for b in bots:
                c = shape_of(b)[1]
                out.append(tds[0][:, c0:c0 + c])
                c0 += c
            return out
        if typ == "Correlation":
            return list(correlation_backward64(l, blobs[bots[0]], blobs[bots[1]], tds[0]))
        if typ == "L1Loss":
            b0 = blobs[bots[0]]
            g0, g1 = l1loss_bwd64(b0, blobs[bots[1]] if len(bots) > 1 else None, float(tds[0].reshape(-1)[0]), **OracleNet._l1_args(l))
            return [g0, g1][:len(bots)]
        raise NotImplementedError("backward of " + typ)
