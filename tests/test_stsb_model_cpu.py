"""CPU: the STS-B oracle (oracle/stsb_ref.py) against the reference's own models.py / fds.py / loss.py (fixture
tests/golden/stsb_model.npz, made by tests/golden/make_golden_stsb_model.py) and against torch's packed nn.LSTM; the
native model's state_dict layout against the fixture's; rnn.LSTM's torch-compatible parameters; and the refusals that
happen before any CUDA call."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import stsb_ref


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stsb_model.npz")


def _golden():
    return np.load(GOLDEN)


def _fixture_oracle(z, dtype=torch.float64):
    """The oracle on the fixture's parameters and batch: (feature, smoothed feature, logits, {kind: loss}, params)."""
    g = lambda k: torch.from_numpy(z[k]).to(dtype)
    p = {"emb": g("p:pair_encoder._text_field_embedder.token_embedder_words.weight").requires_grad_(True),
         "lstm": {k.split(".")[-1]: g(k).requires_grad_(True) for k in z.files
                  if k.startswith("p:pair_encoder._phrase_layer._module.")}}
    W, b = g("p:sts-b_pred_layer.weight").requires_grad_(True), g("p:sts-b_pred_layer.bias").requires_grad_(True)
    s1, s2 = torch.from_numpy(z["s1"]), torch.from_numpy(z["s2"])
    B, T1, T2 = s1.shape[0], s1.shape[1], s2.shape[1]
    T = max(T1, T2)
    ids = torch.cat([torch.nn.functional.pad(s1, (0, T - T1)), torch.nn.functional.pad(s2, (0, T - T2))])
    lens = torch.cat([(s1 != 0).sum(1), (s2 != 0).sum(1)])
    feat = stsb_ref.forward(p, ids, lens, B)
    tables = {k: g(f"p:FDS.{k}") for k in ("running_mean_last_epoch", "running_var_last_epoch",
                                            "smoothed_mean_last_epoch", "smoothed_var_last_epoch")}
    label, weight = g("label"), g("weight")
    fs = stsb_ref.fds_smooth(feat, label, tables)
    logits = fs @ W.t() + b
    losses = {k: stsb_ref.loss(k, logits, label / 5, weight) for k in ("mse", "l1", "focal_mse", "focal_l1", "huber")}
    return feat, fs, logits, losses, dict(p["lstm"], emb=p["emb"], W=W, b=b)


def test_oracle_matches_reference_fixture():
    """Feature, FDS-smoothed embs, logits, every loss kind and every parameter gradient of the reference's own model
    (fp32) against the float64 oracle, to fp32 tolerance."""
    z = _golden()
    feat, fs, logits, losses, p = _fixture_oracle(z)
    close = lambda got, want, tol=2e-5: np.abs(got - want).max() <= tol * max(1.0, np.abs(want).max())
    assert close(feat.detach().numpy(), z["feature"])
    assert close(fs.detach().numpy(), z["embs"])
    assert close(logits.detach().numpy(), z["logits"])
    for k, v in losses.items():
        assert abs(v.item() - float(z[f"loss_{k}"])) <= 2e-5 * abs(float(z[f"loss_{k}"])) + 1e-7, k
    assert float(z["loss"]) == float(z["loss_mse"])
    losses["mse"].backward()
    names = {"emb": "pair_encoder._text_field_embedder.token_embedder_words.weight", "W": "sts-b_pred_layer.weight",
             "b": "sts-b_pred_layer.bias"}
    for k, t in p.items():
        want = z["g:" + names.get(k, f"pair_encoder._phrase_layer._module.{k}")]
        got = t.grad.numpy()
        assert np.abs(got - want).max() <= 1e-4 * np.abs(want).max() + 1e-9, k
    # the padding row of the embedding gets no gradient, and the reference zeroes its weight
    assert not z["g:pair_encoder._text_field_embedder.token_embedder_words.weight"][0].any()
    assert not z["p:pair_encoder._text_field_embedder.token_embedder_words.weight"][0].any()


def _native_args(fds):
    return SimpleNamespace(d_word=24, n_layers_highway=0, glove=1, train_words=1, d_hid=20, n_layers_enc=2,
                           dropout=0.0, fds=fds, bucket_num=50, bucket_start=0, start_update=0, start_smooth=1,
                           fds_kernel='gaussian', fds_ks=5, fds_sigma=2, fds_mmt=0.9, cuda=-1, loss='mse',
                           huber_beta=0.5)


class _Vocab:
    def get_vocab_size(self, ns):
        return 37

    def get_token_index(self, tok):
        return 0


class _Task:
    name = 'sts-b'


@pytest.mark.parametrize("fds", [1, 0], ids=["fds", "nofds"])
def test_native_state_dict_matches_reference(fds):
    """Keys, order and shapes of the native model's state_dict equal the reference model's; the fixture loads into
    it (strict) and comes back unchanged."""
    import models
    z = _golden()
    m = models.build_model(_native_args(fds), _Vocab(), torch.randn(37, 24), [_Task()])
    sd = m.state_dict()
    sfx = "" if fds else "_nofds"
    assert list(sd) == list(z["names" + sfx])
    assert [str(tuple(v.shape)) for v in sd.values()] == list(z["shapes" + sfx])
    # the padding row is zero, as AllenNLP's Embedding makes it
    assert not sd["pair_encoder._text_field_embedder.token_embedder_words.weight"][0].any()
    if fds:
        m.load_state_dict({k: torch.from_numpy(np.asarray(z["p:" + k])) for k in sd}, strict=True)
        for k, v in m.state_dict().items():
            assert np.array_equal(v.numpy(), z["p:" + k]), k


def _packed_reference(lstm, emb, ids, lens):
    x = emb[ids]
    pk = torch.nn.utils.rnn.pack_padded_sequence(x, lens, batch_first=True, enforce_sorted=False)
    o, _ = lstm(pk)
    o, _ = torch.nn.utils.rnn.pad_packed_sequence(o, batch_first=True, total_length=ids.shape[1])
    return o


def test_oracle_matches_packed_torch_lstm():
    torch.manual_seed(0)
    B, T1, T2, V, D, H = 5, 7, 9, 37, 24, 20
    lstm = torch.nn.LSTM(D, H, 2, bidirectional=True, batch_first=True).double()
    emb = torch.randn(V, D, dtype=torch.float64)
    l1 = torch.tensor([7, 1, 3, 5, 2])
    l2 = torch.tensor([9, 4, 1, 6, 8])
    s1 = torch.randint(1, V, (B, T1)) * (torch.arange(T1)[None] < l1[:, None])
    s2 = torch.randint(1, V, (B, T2)) * (torch.arange(T2)[None] < l2[:, None])
    u = _packed_reference(lstm, emb, s1, l1).masked_fill(~(torch.arange(T1)[None] < l1[:, None])[..., None],
                                                          float("-inf")).max(1).values
    v = _packed_reference(lstm, emb, s2, l2).masked_fill(~(torch.arange(T2)[None] < l2[:, None])[..., None],
                                                          float("-inf")).max(1).values
    want = torch.cat([u, v, (u - v).abs(), u * v], 1)
    T = max(T1, T2)
    ids = torch.cat([torch.nn.functional.pad(s1, (0, T - T1)), torch.nn.functional.pad(s2, (0, T - T2))])
    p = {"emb": emb, "lstm": dict(lstm.named_parameters())}
    got = stsb_ref.forward(p, ids, torch.cat([l1, l2]), B)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


def test_rnn_lstm_parameters_are_torch_lstm():
    import rnn
    torch.manual_seed(3)
    mine = rnn.LSTM(300, 1500, 2, bidirectional=True, batch_first=True)
    torch.manual_seed(3)
    ref = torch.nn.LSTM(300, 1500, 2, bidirectional=True, batch_first=True)
    a, b = mine.state_dict(), ref.state_dict()
    assert list(a) == list(b)
    assert all(torch.equal(a[k], b[k]) for k in a)
    assert mine.hidden_p == 1536 and mine.input_p == 320
    ref.load_state_dict(a)
    mine.load_state_dict(ref.state_dict())


def test_refusals_before_cuda():
    import _lib
    import models
    from types import SimpleNamespace
    args = SimpleNamespace(d_word=24, n_layers_highway=1, glove=0, train_words=0, d_hid=20, n_layers_enc=2,
                           dropout=0.2, fds=0, cuda=-1)
    with pytest.raises(ValueError, match="n_layers_highway"):
        models.build_model(args, None, None, [])
    raw = _lib.raw
    # null pointers, bad sizes and steps are refused on the host
    assert raw("dirb200_lstm_fwd_step")(None, None, None, None, 4, 2, 64, 1, 0, None, None, None, None, None) == -1
    assert "null" in _lib.last_error()
    p = _lib.c_void_p(16)
    assert raw("dirb200_lstm_layer_fwd")(p, p, p, p, 5000, 2, 64, 1, p, p, p, p, None) == -1
    assert "T must be" in _lib.last_error()
    assert raw("dirb200_lstm_layer_fwd")(p, p, p, p, 4, 2, 100, 1, p, p, p, p, None) == -1
    assert "Hp" in _lib.last_error()
    assert raw("dirb200_lstm_fwd_step")(p, p, p, p, 4, 2, 64, 1, 4, p, p, p, p, None) == -1
    assert "step" in _lib.last_error()
    assert raw("dirb200_lstm_layer_fwd")(p, p, p, p, 4, 2, 64, 1, p, p, None, p, None) == -1
    assert "gates" in _lib.last_error()
    assert raw("dirb200_lstm_bwd_step")(p, p, p, p, p, 4, 0, 64, 0, p, p, p, None) == -1
    # the whole-layer backward: every pointer, then T, M and Hp
    for k in range(8):
        args = [p] * 8
        args[k] = None
        assert raw("dirb200_lstm_layer_bwd")(*args[:5], 4, 2, 64, *args[5:], None) == -1, k
        assert "lstm_layer_bwd: null" in _lib.last_error()
    for T, M, Hp, what in [(0, 2, 64, "T must be"), (4097, 2, 64, "T must be"), (4, 0, 64, "M must be"),
                           (4, 65536, 64, "M must be"), (4, 2, 0, "Hp"), (4, 2, 100, "Hp"), (4, 2, 4160, "Hp")]:
        assert raw("dirb200_lstm_layer_bwd")(p, p, p, p, p, T, M, Hp, p, p, p, None) == -1, (T, M, Hp)
        assert what in _lib.last_error() and "lstm_layer_bwd" in _lib.last_error()
    assert raw("dirb200_pair_maxpool_fwd")(p, p, None, 2, 0, 20, 64, p, p, None) == -1
    assert raw("dirb200_embed_gather")(p, p, p, None, 37, 4, 3, 24, 32, p, None) == -1
    assert raw("dirb200_lstm_prep_weights")(p, p, p, p, p, p, p, p, 20, 24, 3, 64, 64, p, p, p, p, p, None) == -1
    assert raw("dirb200_col_sum_bf16")(None, 4, 4, p, None) == -1
