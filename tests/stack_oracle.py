"""OracleNet with Caffe's need-backward pruning (the reference's net.cpp:120-170), for the stacked FlowNet2 training graphs.

OracleNet.backward differentiates every layer under a loss.  On a stage trained on frozen predecessors that walks into the warp
block and stops at ChannelNorm, which has no backward.  Caffe instead decides once, from the graph, which layers need backward:
a layer does when it has a parameter with lr_mult != 0 (default 1) or a bottom that carries a gradient, and its type allows
backward; a bottom receives a gradient only if it carries one and its propagate_down is not false.  A layer whose parameters all
have lr_mult 0 reports no parameter gradient.  This is the rule of the engine's Net::NeedBackward, restated independently over
the oracle's own parse.
"""
from oracle.net import OracleNet, get, getall

# layers whose AllowBackward() is false in the reference (resample_layer.hpp:25, data_augmentation_layer.hpp:29, the two
# augmentation-parameter layers, downsample_layer.cu:131-137)
NO_BACKWARD = ("Resample", "DataAugmentation", "FlowAugmentation", "GenerateAugmentationParameters", "Downsample")


def lr_mults(l):
    """lr_mult of each parameter blob of a layer (ParamSpec default 1); only convolutions have parameters in these graphs."""
    if get(l, "type") not in ("Convolution", "Deconvolution"):
        return []
    specs = getall(l, "param")
    n = 2 if get(get(l, "convolution_param", []), "bias_term", "true") == "true" else 1
    return [float(get(specs[i], "lr_mult", 1)) if i < len(specs) else 1.0 for i in range(n)]


class PrunedOracleNet(OracleNet):
    def __init__(self, *args, **kwargs):
        super(PrunedOracleNet, self).__init__(*args, **kwargs)
        blob_need = {n: get(self.root, "force_backward", "false") == "true" for n in self.input_names}
        self.layer_need = {}
        for l in self.layers:
            typ = get(l, "type")
            need = any(lr != 0 for lr in lr_mults(l)) or any(blob_need.get(b, False) for b in getall(l, "bottom"))
            need = need and typ not in NO_BACKWARD
            self.layer_need[get(l, "name")] = need
            for t in getall(l, "top"):
                blob_need[t] = need or blob_need.get(t, False)
        self.blob_need = blob_need

    def backward_layer(self, l, bots, tops, tds, P):
        name = get(l, "name")
        names = getall(l, "bottom")
        if not self.layer_need[name]:
            return [None] * len(bots)
        grads = super(PrunedOracleNet, self).backward_layer(l, bots, tops, tds, P)
        pd = getall(l, "propagate_down")
        grads = [g if self.blob_need.get(b, False) and not (i < len(pd) and pd[i] == "false") else None
                 for i, (b, g) in enumerate(zip(names, grads))]
        lrs = lr_mults(l)
        if name in P and lrs and all(lr == 0 for lr in lrs):
            del P[name]
        return grads
