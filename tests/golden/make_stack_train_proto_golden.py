"""Parses the authored training prototxts of the stacked FlowNet2 schedule (models/FlowNet2-CS_train, -CSS_train, -SD_train and
FlowNet2_train .prototxt.template) with the REFERENCE's own caffe_pb2 (python/caffe/proto/caffe_pb2.py: any field that is not in
the reference's caffe.proto makes text_format.Merge raise) and writes what it read to tests/golden/ref_pb2_stack_train_prototxt.json,
against which the engine's parser is checked.  Same fields as make_train_proto_golden.py, plus every layer's ParamSpecs
(lr_mult, decay_mult: the frozen predecessors).  Run in the container that has /root/reference:
    PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION=python python tests/golden/make_stack_train_proto_golden.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, "/root/reference/python/caffe/proto")

STAGES = ("FlowNet2-CS", "FlowNet2-CSS", "FlowNet2-SD", "FlowNet2")


def read(caffe_pb2, text_format, txt):
    net = caffe_pb2.NetParameter()
    text_format.Merge(txt, net)
    layers = []
    for l in net.layer:
        e = {"name": l.name, "type": l.type, "bottom": list(l.bottom), "top": list(l.top), "loss_weight": [float(x) for x in l.loss_weight],
             "propagate_down": [bool(x) for x in l.propagate_down],
             "param": [[float(p.lr_mult), float(p.decay_mult)] for p in l.param]}
        if l.type == "L1Loss":
            p = l.l1_loss_param
            e["l1"] = [p.l2_per_location, p.l2_prescale_by_channels, p.normalize_by_num_entries, float(p.epsilon), float(p.plateau)]
        if l.type in ("Convolution", "Deconvolution"):
            c = l.convolution_param
            e["conv"] = [c.num_output, list(c.kernel_size), list(c.stride), list(c.pad)]
        if l.type == "Eltwise":
            e["coeff"] = [float(x) for x in l.eltwise_param.coeff]
        if l.HasField("augmentation_param"):
            a = l.augmentation_param
            e["aug"] = {"crop": [a.crop_width, a.crop_height], "mode": a.mode}
        if l.type == "Input":
            e["shapes"] = [list(s.dim) for s in l.input_param.shape]
        layers.append(e)
    return {"name": net.name, "layers": layers}


def main():
    import caffe_pb2
    from google.protobuf import text_format
    import flownet2_b200 as F
    out = {s: read(caffe_pb2, text_format, F.fill_train_template(F.train_template(s), 448, 320, 512, 384, 8)) for s in STAGES}
    with open(os.path.join(HERE, "ref_pb2_stack_train_prototxt.json"), "w") as f:
        json.dump(out, f)
    print("wrote", {s: len(v["layers"]) for s, v in out.items()})


if __name__ == "__main__":
    main()
