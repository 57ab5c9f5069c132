"""CPU oracle of the reference's latency/ deployment network (latency/operations.py, latency/model_seg.py): the train/ restatement
of fasterseg_oracle.py with nearest resizes and the single-conv stride-2 FactorizedReduce.  Pure torch CPU, fp32 with the same
fp16 storage rounding (_q) as fasterseg_oracle.py.  Pinned to tests/golden/latency_variant.npz (oracle/make_golden_latency_variant.py)."""
from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

from oracle import fasterseg_oracle as orc
from oracle.fasterseg_oracle import Params, _q, conv2d, conv_norm, feature_fusion, head


def nearest_index(n_in, n_out):
    """torch's legacy 'nearest' source index per output index: min(floor(dst * (float32(in) / float32(out))), in - 1) in fp32"""
    scale = np.float32(n_in) / np.float32(n_out)
    src = np.floor(np.arange(n_out, dtype=np.float32) * scale).astype(np.int64)
    return torch.from_numpy(np.minimum(src, n_in - 1))


def nearest(x, size):
    """F.interpolate(x, size, mode='nearest'), written out"""
    Ho, Wo = int(size[0]), int(size[1])
    return x.index_select(2, nearest_index(x.shape[2], Ho)).index_select(3, nearest_index(x.shape[3], Wo))


def basic_residual_downup_1x(x, p: Params, stride=1, training=False):
    """latency/operations.py:264-271"""
    H, W = x.shape[2], x.shape[3]
    y = conv2d(nearest(x, (H // 2, W // 2)), p["conv1.weight"], None, 1, 1)
    y = orc._bn(y, p.sub("bn1"), False)
    if stride == 1:
        y = nearest(_q(y), (H, W))
    return _q(F.relu(y))


def basic_residual_downup_2x(x, p: Params, stride=1, training=False):
    """latency/operations.py:426-436"""
    H, W = x.shape[2], x.shape[3]
    y = _q(F.relu(orc._bn(conv2d(nearest(x, (H // 2, W // 2)), p["conv1.weight"], None, 1, 1), p.sub("bn1"), False)))
    y = orc._bn(conv2d(y, p["conv2.weight"], None, 1, 1), p.sub("bn2"), False)
    if stride == 1:
        y = nearest(_q(y), (H, W))
    return _q(F.relu(y))


def factorized_reduce(x, p: Params, stride=1, training=False):
    """latency/operations.py:510-520 (non-slimmable): stride 2 = one 1x1 stride-2 conv C_in -> C_out -> BN -> ReLU"""
    if stride == 2:
        return _q(F.relu(orc._bn(conv2d(x, p["conv1.weight"], None, 2, 0), p.sub("bn"), False)))
    return x


OP_FUNCS = [factorized_reduce, orc.basic_residual_1x, basic_residual_downup_1x, orc.basic_residual_2x, basic_residual_downup_2x]


def student_forward(x, sd: Dict[str, torch.Tensor], st: orc.StudentStructure, return_pred8_lowres=False):
    """eval forward of latency/model_seg.py:298-366 -> logits upsampled x8 (nearest), shape (N, 19, H, W)"""
    P = Params(sd)
    H = x.shape[2]
    y = conv_norm(x, P.sub("stem.0"), 3, 2, 1, False)
    y = orc.basic_residual_2x(y, P.sub("stem.1"), 2, False)
    y = orc.basic_residual_2x(y, P.sub("stem.2"), 2, False)
    nb = st.branch
    outputs = [y] * nb
    taps = {8: [y] * nb, 16: [y] * nb, 32: [y] * nb}
    for layer, groups in enumerate(st.branch_groups):
        for g in groups:
            spec = st.cells["%d-%d" % (layer, g[0])]
            o = OP_FUNCS[spec.op](outputs[g[0]], P.sub("cells.%d-%d._op._op" % (layer, g[0])), 2 if spec.down else 1)
            scale = int(H // o.shape[2])
            for b in g:
                outputs[b] = o
                if scale in taps:
                    taps[scale][b] = o

    def arm_refine(coarse, arm, refine, skip):
        o = conv_norm(coarse, P.sub(arm), 1, 1, 0, False)
        o = _q(nearest(o, (o.shape[2] * 2, o.shape[3] * 2)))   # twice the coarse map (latency/model_seg.py:305,309,315)
        return conv_norm(torch.cat([o, skip], 1), P.sub(refine), 3, 1, 1, False)

    pred8 = []
    for b in range(nb):
        last = st.lasts[b]
        if last == 2:
            o = arm_refine(taps[32][b], "arms32.0", "refines32.0", taps[16][b])
            pred8.append(arm_refine(o, "arms32.1", "refines32.1", taps[8][b]))
        elif last == 1:
            pred8.append(arm_refine(taps[16][b], "arms16", "refines16", taps[8][b]))
        else:
            pred8.append(taps[8][b])
    p8 = head(feature_fusion(torch.cat(pred8, 1), P.sub("ffm"), False), P.sub("heads8"), False)
    if return_pred8_lowres:
        return p8
    return nearest(p8, (p8.shape[2] * 8, p8.shape[3] * 8))
