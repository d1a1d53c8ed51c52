"""Shared by the TransformNet recurrence fixture (tests/golden/make_golden_convlstm_state.py) and its tests: the
inputs, regenerated from a seed; the float CPU restatement of TransformNet.forward with a carried ConvLSTM state
(built on oracle/stage2_oracle.py's layers), pinned bit for bit against the reference by the fixture's generator; and
the fixture's compact form of an output tensor."""
import torch
import torch.nn.functional as F

from oracle import stage2_oracle as SO

NF, FRAMES, H, W = 32, 4, 64, 96
SAMPLE_STRIDE = 17                    # the fixture keeps every 17th element of each output (and its float64 sums)


def recurrence_inputs(seed, frames=FRAMES, h=H, w=W, nf=NF):
    """Frames of a recurrence, the input of the random-state step and that state (hidden, cell): hidden uniform in
    [-3, 3], cell normal with std 3, so the gates and the cell leave the linear region of sigmoid / tanh."""
    g = torch.Generator().manual_seed(seed)
    xs = [torch.rand(1, 12, h, w, generator=g) for _ in range(frames)]
    x_r = torch.rand(1, 12, h, w, generator=g)
    c = 4 * nf
    h0 = (torch.rand(1, c, h // 4, w // 4, generator=g) * 2 - 1) * 3
    c0 = torch.randn(1, c, h // 4, w // 4, generator=g) * 3
    return xs, x_r, (h0, c0)


def transformnet_forward_state(sd, X, prev_state, blocks=5):
    """TransformNet.forward (network_local.py:88-115) with ConvLSTM.forward's prev_state = (hidden, cell)
    (network_local.py:18-53): cell = sigmoid(r) * prev_cell + sigmoid(i) * tanh(g).  Returns (Y, hidden, cell)."""
    lrelu = lambda t: F.leaky_relu(t, 0.2)
    e1a = lrelu(SO._rconv(sd, "conv1a", X[:, :6], 7))
    e1b = lrelu(SO._rconv(sd, "conv1b", X[:, 6:], 7))
    e2a = lrelu(SO._rconv(sd, "conv2a", e1a, 3, 2))
    e2b = lrelu(SO._rconv(sd, "conv2b", e1b, 3, 2))
    rb = lrelu(SO._rconv(sd, "conv3", torch.cat((e2a, e2b), 1), 3, 2))
    for b in range(blocks):
        t = lrelu(SO._rconv(sd, f"ResBlocks.{b}.conv1", rb, 3))
        rb = SO._rconv(sd, f"ResBlocks.{b}.conv2", t, 3) + rb
    hidden0, cell0 = prev_state
    gates = F.conv2d(torch.cat((rb, hidden0), 1), sd["convlstm.Gates.weight"], sd["convlstm.Gates.bias"], padding=1)
    i_g, r_g, o_g, c_g = gates.chunk(4, 1)
    cell = torch.sigmoid(r_g) * cell0 + torch.sigmoid(i_g) * torch.tanh(c_g)
    hidden = torch.sigmoid(o_g) * torch.tanh(cell)
    d2 = lrelu(SO._rconv(sd, "deconv1", hidden, 3, upsample=2))
    d1 = lrelu(SO._rconv(sd, "deconv2", torch.cat((d2, e2a), 1), 3, upsample=2))
    y = torch.tanh(SO._rconv(sd, "deconv3", torch.cat((d1, e1a), 1), 7))
    return y, hidden, cell


def recurrence(sd, xs, state=None):
    """Runs the frames in order, each call fed the previous call's state (None: zero state, the stateless oracle).
    Returns the per-frame outputs Y and the last state."""
    ys = []
    for x in xs:
        y, h, c = SO.transformnet_forward(sd, x) if state is None else transformnet_forward_state(sd, x, state)
        ys.append(y)
        state = (h, c)
    return ys, state


def digest(t):
    """What the fixture keeps of an output: every SAMPLE_STRIDE-th element and the float64 sum and absolute sum."""
    flat = t.detach().reshape(-1)
    return {"sample": flat[::SAMPLE_STRIDE].clone(), "sum": flat.double().sum(), "abs_sum": flat.double().abs().sum()}
