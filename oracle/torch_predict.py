"""ORACLE (test infrastructure) — plain-PyTorch functional restatement of the eval-mode prediction stage.

Only tests/ and tools/ may import this.  Like oracle/torch_dense.py, every function takes a module that carries the
reference's parameter tree (the reference's own module or the drop-in module of stp3_b200) and evaluates the
reference's eval-mode equations with torch.nn.functional ops in the dtype of the input (fp64 for the oracle, fp32 for
the torch eager baseline of tools/predict_bench.py).  Nothing here calls the modules' own forward().

  Bottleneck(downsample) / DistributionModule   stp3/layers/convolutions.py:65-170, stp3/models/distributions.py
  LayerNorm / Block / Bottleblock               stp3/layers/convolutions.py:283-380
  SpatialGRU / Dual_GRU                         stp3/layers/temporal.py:11-160
  FuturePrediction                              stp3/models/future_prediction.py
  the stage between temporal model and decoder  stp3/models/stp3.py:157-176, 320-352
"""
import torch
import torch.nn.functional as F

from .torch_dense import _bn, decoder, deeplab_head


def _w(p, x):
    return None if p is None else p.to(x.dtype)


def _conv(x, conv, **kw):
    return F.conv2d(x, _w(conv.weight, x), _w(conv.bias, x), stride=conv.stride, padding=conv.padding,
                    groups=conv.groups, **kw)


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / 2 ** 0.5))


def layer_norm_cf(x, ln):
    """Channels-first LayerNorm over dim 1 (biased variance)."""
    u = x.mean(1, keepdim=True)
    s = (x - u).pow(2).mean(1, keepdim=True)
    x = (x - u) / torch.sqrt(s + ln.eps)
    return _w(ln.weight, x)[:, None, None] * x + _w(ln.bias, x)[:, None, None]


def maxpool2_pad(x):
    """The downsampling Bottleneck's skip input: zero-pad an odd H / W at the bottom / right, then MaxPool 2x2."""
    x = F.pad(x, (0, x.shape[-1] % 2, 0, x.shape[-2] % 2), value=0)
    return F.max_pool2d(x, 2, 2)


def bottleneck(x, m):
    L = m.layers
    y = F.relu(_bn(_conv(x, L.conv_down_project), L.abn_down_project[0]))
    y = F.relu(_bn(_conv(y, L.conv), L.abn[0]))
    y = F.relu(_bn(_conv(y, L.conv_up_project), L.abn_up_project[0]))
    p = m.projection
    return y + _bn(_conv(maxpool2_pad(x), p.conv_skip_proj), p.bn_skip_proj)


def distribution(x, m):
    """x (B, 1, C, H, W) -> (B, 1, 2 * latent) mu | log sigma."""
    y = x[:, 0]
    for b in m.encoder.model:
        y = bottleneck(y, b)
    y = _conv(y.mean(dim=(2, 3), keepdim=True), m.decoder[1])
    return y.view(x.shape[0], 1, -1)


def block(x, m):
    """ConvNeXt Block."""
    y = _conv(x, m.dwconv).permute(0, 2, 3, 1)
    y = F.layer_norm(y, m.norm.normalized_shape, _w(m.norm.weight, y), _w(m.norm.bias, y), m.norm.eps)
    y = F.linear(y, _w(m.pwconv1.weight, y), _w(m.pwconv1.bias, y))
    y = F.linear(_gelu(y), _w(m.pwconv2.weight, y), _w(m.pwconv2.bias, y))
    if m.gamma is not None:
        y = _w(m.gamma, y) * y
    return x + y.permute(0, 3, 1, 2)


def bottleblock(x, m):
    L = m.layers
    y = x
    for i in (0, 3, 6):
        y = _gelu(layer_norm_cf(_conv(y, L[i]), L[i + 1]))
    return y + (_gelu(_conv(x, m.projection[0])) if m.projection is not None else x)


def _gru_cell(x, h, cu, cr, ct):
    xh = torch.cat([x, h], 1)
    u = torch.sigmoid(_conv(xh, cu))
    r = torch.sigmoid(_conv(xh, cr))
    ht = _conv(torch.cat([x, (1.0 - r) * h], 1), ct)
    return (1.0 - u) * h + u * ht


def spatial_gru(x, h, m):
    """x (B, T, C, H, W), h (B, hidden, H, W) -> (B, T, C, H, W)."""
    outs = []
    for t in range(x.shape[1]):
        h = _gru_cell(x[:, t], h, m.conv_update, m.conv_reset, m.conv_state_tilde)
        outs.append(_conv(h, m.conv_decoder))
    return torch.stack(outs, 1)


def dual_gru(x, state, m):
    """x (B, 1, latent, H, W), state (B, S, hidden, H, W) -> (B, n_future, hidden, H, W)."""
    cell1 = lambda a, h: _gru_cell(a, h, m.conv_update_1, m.conv_reset_1, m.conv_state_tilde_1)
    cell2 = lambda a, h: _gru_cell(a, h, m.conv_update_2, m.conv_reset_2, m.conv_state_tilde_2)
    h = state[:, 0]
    for t in range(state.shape[1] - 1):
        h = cell2(state[:, t], h)
    s1 = s2 = state[:, -1]
    x = x[:, 0]
    preds = []
    for _ in range(m.n_future):
        s1 = cell1(x, s1)
        h = cell2(s2, h)
        s2 = _conv(h, m.conv_decoder_2)
        g = torch.softmax(_conv(bottleblock(torch.cat([s1, s2], 1), m.trusting_gate[0]), m.trusting_gate[1]), dim=1)
        cur = s2 * g[:, 0:1] + s1 * g[:, 1:]
        preds.append(cur)
        if m.mixture:
            s1 = s2 = cur
    return torch.stack(preds, 1)


def _frames(x, fn):
    b, s = x.shape[:2]
    y = fn(x.reshape(b * s, *x.shape[2:]))
    return y.view(b, s, *y.shape[1:])


def _seq(x, seq):
    for blk in seq:
        x = block(x, blk)
    return x


def future_prediction(x, state, m):
    """x (B, 1, latent, H, W), state (B, S, C, H, W) -> (B, S + n_future, C, H, W)."""
    y = dual_gru(x, state, m.dual_grus)
    y = _frames(y, lambda v: _seq(v, m.res_blocks1))
    y = torch.cat([state, y], 1)
    h0 = y[:, 0]
    for i in range(m.n_spatial_gru):
        y = spatial_gru(y, h0, m.spatial_grus[i])
        rb = m.res_blocks[i]
        y = _frames(y, (lambda v, rb=rb: deeplab_head(v, rb)) if i == m.n_spatial_gru - 1 else
                    (lambda v, rb=rb: _seq(v, rb)))
    return y


def predict_stage(states, model):
    """STP3's stage between the temporal model and the decoder in eval mode: the sample is mu (zero noise) broadcast
    over the map, or zeros without PROBABILISTIC.  states (B, S, C, H, W) -> (B, S + n_future, C, H, W)."""
    b, s, _, h, w = states.shape
    lat = model.latent_dim
    if model.cfg.PROBABILISTIC.ENABLED:
        mu = distribution(states[:, -1:], model.present_distribution)[:, :, :lat]
        x = mu.view(b, 1, lat, 1, 1).expand(b, 1, lat, h, w)
    else:
        x = states.new_zeros(b, 1, lat, h, w)
    return future_prediction(x, states, model.future_prediction)


def predict_and_decode(states, model):
    """predict_stage -> Decoder: the dict of the reference's decoder outputs over all frames."""
    return decoder(predict_stage(states, model), model.decoder)
