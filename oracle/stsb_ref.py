"""STS-B-DIR's sentence-pair model (sts-b-dir/models.py:116-166 with AllenNLP 0.5's Embedding, the 'lstm' seq2seq
wrapper and get_text_field_mask restated) as a pure torch function of a parameter dict -- TEST INFRASTRUCTURE ONLY
(see oracle/dir_oracle.py for the rules).  Any float dtype; dropout arrives as explicit multipliers (keep / (1 - p)).

Parameter keys are the reference model's state_dict keys without the 'pair_encoder.' prefix handling: `emb` is
_text_field_embedder.token_embedder_words.weight, `lstm` the phrase layer's torch.nn.LSTM keys (weight_ih_l0, ...).

`force(k, d, s, h, c) -> (h, c)`, when given, replaces the state entering step s of direction d of layer k (rows in the
order of `lens`): the teacher-forcing hook the GPU tests use to compare one step of the native recurrence at a time.
"""
import torch


def cell(x_proj, h, c, w_hh, b):
    """One LSTM step: gates (i, f, g, o) = x_proj + h . w_hh^T + b."""
    a = x_proj + h @ w_hh.t() + b
    i, f, g, o = a.chunk(4, dim=-1)
    i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
    c2 = f * c + i * g
    return o * torch.tanh(c2), c2


def lstm_layer(lstm, k, x, lens, force=None):
    """x [M, T, Din] batch-first, lens [M] (>= 1) -> [M, T, 2H], zeros at t >= lens (packed semantics)."""
    M, T, _ = x.shape
    outs = []
    for d, sfx in enumerate(("", "_reverse")):
        w_ih, w_hh = lstm[f"weight_ih_l{k}{sfx}"], lstm[f"weight_hh_l{k}{sfx}"]
        b = lstm[f"bias_ih_l{k}{sfx}"] + lstm[f"bias_hh_l{k}{sfx}"]
        H = w_hh.shape[1]
        xp = x @ w_ih.t()
        h = x.new_zeros(M, H)
        c = x.new_zeros(M, H)
        y = x.new_zeros(M, T, H)
        rows = torch.arange(M)
        for s in range(T):
            active = s < lens
            if not bool(active.any()):
                break
            if force is not None:
                h, c = force(k, d, s, h, c)
            tau = torch.where(active, s if d == 0 else lens - 1 - s, torch.zeros_like(lens))
            h2, c2 = cell(xp[rows, tau], h, c, w_hh, b)
            keep = active[:, None]
            h = torch.where(keep, h2, torch.zeros_like(h2))
            c = torch.where(keep, c2, torch.zeros_like(c2))
            y = y.index_put((rows[active], tau[active]), h[active])
        outs.append(y)
    return torch.cat(outs, dim=-1)


def encode(p, ids, lens, dmul_emb=None, force=None):
    """ids [M, T] int64, lens [M] -> the last LSTM layer's output [M, T, 2H] (dmul_emb: [M, T, d_word] or None)."""
    x = p["emb"][ids]
    x = x * (torch.arange(ids.shape[1])[None, :] < lens[:, None])[..., None].to(x.dtype)
    if dmul_emb is not None:
        x = x * dmul_emb
    k = 0
    while f"weight_ih_l{k}" in p["lstm"]:
        x = lstm_layer(p["lstm"], k, x, lens, force)
        k += 1
    return x


def pair_features(enc, lens, B, dmul_out=None, arg=None):
    """enc [2B, T, 2H] (s1 rows then s2 rows) -> [B, 8H]: masked max over time, then [u, v, |u - v|, u * v].
    arg [2B, 2H], when given, names the time each maximum is taken from (to follow another implementation's choice
    among near-ties, so that the gradient flows to the same positions)."""
    if dmul_out is not None:
        enc = enc * dmul_out
    if arg is not None:
        m = enc.gather(1, arg.long()[:, None, :]).squeeze(1)
    else:
        mask = torch.arange(enc.shape[1])[None, :] < lens[:, None]
        m, _ = enc.masked_fill(~mask[..., None], float("-inf")).max(dim=1)
    u, v = m[:B], m[B:]
    return torch.cat([u, v, torch.abs(u - v), u * v], 1)


def bucket(label, bucket_num=50, bucket_start=0):
    """sts-b-dir/fds.py:51-57: the np.histogram bin of label over [0, 5] (5 itself in the last bin)."""
    import numpy as np
    label = np.float32(label)
    _, edges = np.histogram(a=np.array([], dtype=np.float32), bins=bucket_num, range=(0., 5.))
    if label == 5.:
        return bucket_num - 1
    return max(np.where(edges > label)[0][0] - 1, bucket_start)


def fds_smooth(feat, labels, tables, bucket_num=50, bucket_start=0, clip=(0.5, 2.0)):
    """FDS.smooth of sts-b-dir/fds.py:128-143 with util.calibrate_mean_var (every variance positive):
    (x - m1[b]) * sqrt(clamp(v2[b] / v1[b], clip)) + m2[b], b the row's bucket.  `tables`: the *_last_epoch
    buffers by name."""
    b = torch.tensor([bucket(float(v), bucket_num, bucket_start) - bucket_start for v in labels.reshape(-1)])
    m1, v1 = tables["running_mean_last_epoch"][b], tables["running_var_last_epoch"][b]
    m2, v2 = tables["smoothed_mean_last_epoch"][b], tables["smoothed_var_last_epoch"][b]
    return (feat - m1) * torch.sqrt(torch.clamp(v2 / v1, *clip)) + m2


def loss(kind, logits, targets, weights=None, huber_beta=0.5, beta=20., gamma=1):
    """sts-b-dir/loss.py's weighted losses with STS-B's defaults (focal: sigmoid, beta 20)."""
    d = (logits - targets).abs()
    if kind == 'mse':
        v = d ** 2
    elif kind == 'l1':
        v = d
    elif kind == 'huber':
        v = torch.where(d < huber_beta, 0.5 * d ** 2 / huber_beta, d - 0.5 * huber_beta)
    else:
        v = (d ** 2 if kind == 'focal_mse' else d) * (2 * torch.sigmoid(beta * d) - 1) ** gamma
    if weights is not None:
        v = v * weights
    return v.mean()


def forward(p, ids, lens, B, dmul_emb=None, dmul_out=None, force=None, arg=None):
    """The pair feature of models.py:137-166 (rows: s1 then s2, padded to a common T)."""
    return pair_features(encode(p, ids, lens, dmul_emb, force), lens, B, dmul_out, arg)
