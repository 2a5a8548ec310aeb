"""Golden fixture for STS-B-DIR's sentence-pair model (sts-b-dir/models.py), produced by running the REFERENCE's own
models.py, fds.py, loss.py and util.py on the CPU in fp32.

Run in the build container only (needs the reference tree, read-only):

    python tests/golden/make_golden_stsb_model.py

The reference imports AllenNLP 0.5, which is not installed; a minimal restatement of the classes models.py uses is
registered under the `allennlp` module names first (test infrastructure, written from AllenNLP 0.5's documented
behaviour):
  Params                      a dict with pop()
  Model                       nn.Module holding the vocabulary
  Highway(d, 0)               the identity (models.py is built with n_layers_highway = 0)
  TimeDistributed(m)          m applied to the [B, T, d] input (identity here)
  util.get_text_field_mask    (ids != 0).long() over the single token field
  InitializerApplicator()     no-op (the default applicator has no initializers)
  BasicTextFieldEmbedder      token embedders registered as token_embedder_{key}, outputs concatenated
  Embedding                   weight [V, d] (given, or xavier_uniform), requires_grad = trainable, row padding_index
                              zeroed, forward = F.embedding(ids, weight, padding_idx=padding_index)
  Seq2SeqEncoder.by_name('lstm').from_params(p)
                              PytorchSeq2SeqWrapper(nn.LSTM(batch_first=True, **p)): lengths = mask.sum(1), sort by
                              length, pack_padded_sequence, run, pad_packed_sequence, zero-pad back to T, restore order
Two torch shims: Tensor.cuda is the identity (models.py:101 and fds.py:49 call .cuda() unconditionally), and
masked_fill_ takes the uint8 mask of models.py:161-162 as bool (torch 2.11 refuses uint8 masks).

Model: d_word 24, d_hid 20, 2 layers, V = 37, dropout 0, GloVe weights given and trainable (--train_words), FDS on
(50 buckets from 0, gaussian ks 5 sigma 2, start_smooth 1) with running_mean_last_epoch = 0.3 N, running_var_last_epoch
= 0.5 + |N|, smoothed_mean_last_epoch = 0.3 N, smoothed_var_last_epoch = 0.5 + |N| (N from torch.manual_seed(5), in that
order, [50, 160] each).  Parameters: torch.manual_seed(0) before build_model (torch's own LSTM / Linear init), GloVe
weights = 0.5 randn(37, 24) drawn first.  Batch B = 5, s1 lengths (7, 1, 3, 5, 2) in T1 = 7, s2 lengths
(9, 4, 1, 6, 8) in T2 = 9, ids from torch.manual_seed(1), labels 5 u (u uniform, seed 2) with label[1] = 5 exactly,
weights 0.5 + u.  Training mode, epoch 1 (FDS smoothing active), loss 'mse'; loss.backward().

Stored:
  s1, s2, label, weight                  inputs
  p:{name}                               every state_dict entry (parameters and FDS buffers) before the step
  names, shapes, names_nofds, shapes_nofds   state_dict keys and shapes with and without FDS
  feature                                the pair encoder's output (before smoothing)
  embs                                   out['embs'] (the same tensor, smoothed in place by FDS.smooth, fds.py:135)
  logits, loss                           out['logits'], out['loss']
  loss_{kind}                            the loss for every --loss kind on the same batch (huber_beta 0.5)
  g:{name}                               every parameter gradient of the 'mse' loss
"""
import os
import sys
import types
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/sts-b-dir"


def _install_allennlp_shim():
    def mod(name):
        m = types.ModuleType(name)
        sys.modules[name] = m
        return m

    class Params(dict):
        pass

    class Model(nn.Module):
        def __init__(self, vocab):
            super().__init__()
            self.vocab = vocab

    class Highway(nn.Module):
        def __init__(self, input_dim, num_layers=1):
            super().__init__()
            assert num_layers == 0
            self._layers = nn.ModuleList()

        def forward(self, x):
            return x

    class TimeDistributed(nn.Module):
        def __init__(self, module):
            super().__init__()
            self._module = module

        def forward(self, x):
            return self._module(x)

    class InitializerApplicator:
        def __call__(self, module):
            pass

    class Embedding(nn.Module):
        def __init__(self, num_embeddings, embedding_dim, weight=None, padding_index=None, trainable=True):
            super().__init__()
            self.output_dim = embedding_dim
            self.padding_index = padding_index
            if weight is None:
                weight = torch.empty(num_embeddings, embedding_dim)
                nn.init.xavier_uniform_(weight)
            self.weight = nn.Parameter(weight.clone(), requires_grad=trainable)
            if padding_index is not None:
                self.weight.data[padding_index].fill_(0)

        def get_output_dim(self):
            return self.output_dim

        def forward(self, ids):
            return F.embedding(ids, self.weight, padding_idx=self.padding_index)

    class BasicTextFieldEmbedder(nn.Module):
        def __init__(self, token_embedders):
            super().__init__()
            self._token_embedders = token_embedders
            for k, e in token_embedders.items():
                self.add_module(f"token_embedder_{k}", e)

        def get_output_dim(self):
            return sum(e.get_output_dim() for e in self._token_embedders.values())

        def forward(self, text_field_input):
            return torch.cat([self._token_embedders[k](text_field_input[k]) for k in sorted(text_field_input)], -1)

    class PytorchSeq2SeqWrapper(nn.Module):
        def __init__(self, module):
            super().__init__()
            self._module = module

        def get_output_dim(self):
            return self._module.hidden_size * (2 if self._module.bidirectional else 1)

        def forward(self, inputs, mask):
            lengths = mask.long().sum(-1)
            order = torch.argsort(lengths, descending=True, stable=True)
            restore = torch.argsort(order)
            pk = nn.utils.rnn.pack_padded_sequence(inputs[order], lengths[order].cpu(), batch_first=True)
            out, _ = self._module(pk)
            out, _ = nn.utils.rnn.pad_packed_sequence(out, batch_first=True)
            T = inputs.shape[1]
            if out.shape[1] < T:
                out = torch.cat([out, out.new_zeros(out.shape[0], T - out.shape[1], out.shape[2])], 1)
            return out[restore]

    class _Lstm:
        @staticmethod
        def from_params(p):
            return PytorchSeq2SeqWrapper(nn.LSTM(batch_first=True, **dict(p)))

    class Seq2SeqEncoder:
        @staticmethod
        def by_name(name):
            assert name == 'lstm'
            return _Lstm

    def get_text_field_mask(text_field_tensors):
        return (text_field_tensors['words'] != 0).long()

    mod("allennlp")
    mod("allennlp.common").Params = Params
    mod("allennlp.models")
    mod("allennlp.models.model").Model = Model
    m = mod("allennlp.modules")
    m.Highway, m.TimeDistributed = Highway, TimeDistributed
    m = mod("allennlp.nn")
    m.util = SimpleNamespace(get_text_field_mask=get_text_field_mask)
    m.InitializerApplicator = InitializerApplicator
    mod("allennlp.modules.text_field_embedders").BasicTextFieldEmbedder = BasicTextFieldEmbedder
    mod("allennlp.modules.token_embedders").Embedding = Embedding
    mod("allennlp.modules.seq2seq_encoders").Seq2SeqEncoder = Seq2SeqEncoder


def _install_torch_shims():
    torch.Tensor.cuda = lambda self, *a, **k: self
    orig = torch.Tensor.masked_fill_

    def masked_fill_(self, mask, value):
        return orig(self, mask.bool() if mask.dtype == torch.uint8 else mask, value)

    torch.Tensor.masked_fill_ = masked_fill_


class Vocab:
    _padding_token = '@@PADDING@@'

    def get_vocab_size(self, namespace):
        return 37

    def get_token_index(self, token):
        return 0


class Task:
    name = 'sts-b'

    def scorer(self, logits, labels):
        pass


def make_args(fds=True, loss='mse'):
    return SimpleNamespace(d_word=24, n_layers_highway=0, glove=1, train_words=1, d_hid=20, n_layers_enc=2,
                           dropout=0.0, fds=fds, bucket_num=50, bucket_start=0, start_update=0, start_smooth=1,
                           fds_kernel='gaussian', fds_ks=5, fds_sigma=2, fds_mmt=0.9, cuda=-1, loss=loss,
                           huber_beta=0.5)


L1, L2 = (7, 1, 3, 5, 2), (9, 4, 1, 6, 8)
T1, T2 = 7, 9


def make_inputs():
    g = torch.Generator().manual_seed(1)
    l1, l2 = torch.tensor(L1), torch.tensor(L2)
    s1 = torch.randint(1, 37, (5, T1), generator=g) * (torch.arange(T1)[None] < l1[:, None])
    s2 = torch.randint(1, 37, (5, T2), generator=g) * (torch.arange(T2)[None] < l2[:, None])
    g = torch.Generator().manual_seed(2)
    label = torch.rand(5, 1, generator=g) * 5
    label[1] = 5.0
    weight = 0.5 + torch.rand(5, 1, generator=g)
    return s1, s2, label, weight


def fds_tables():
    torch.manual_seed(5)
    return {"running_mean_last_epoch": 0.3 * torch.randn(50, 160),
            "running_var_last_epoch": 0.5 + torch.randn(50, 160).abs(),
            "smoothed_mean_last_epoch": 0.3 * torch.randn(50, 160),
            "smoothed_var_last_epoch": 0.5 + torch.randn(50, 160).abs()}


def main():
    _install_allennlp_shim()
    _install_torch_shims()
    sys.path.insert(0, REF)
    import models as ref_models

    def build(fds=True, loss='mse'):
        torch.manual_seed(0)
        embs = 0.5 * torch.randn(37, 24)
        m = ref_models.build_model(make_args(fds, loss), Vocab(), embs, [Task()])
        if fds:
            for k, v in fds_tables().items():
                setattr(m.FDS, k, v.clone())
        return m

    out = {}
    nofds = build(fds=False)
    out["names_nofds"] = np.array(list(nofds.state_dict()))
    out["shapes_nofds"] = np.array([str(tuple(v.shape)) for v in nofds.state_dict().values()])
    model = build()
    sd = model.state_dict()
    out["names"] = np.array(list(sd))
    out["shapes"] = np.array([str(tuple(v.shape)) for v in sd.values()])
    for k, v in sd.items():
        out[f"p:{k}"] = v.detach().numpy().copy()
    s1, s2, label, weight = make_inputs()
    out.update(s1=s1.numpy(), s2=s2.numpy(), label=label.numpy(), weight=weight.numpy())
    model.train()
    seen = {}
    model.pair_encoder.register_forward_hook(lambda mod, inp, o: seen.__setitem__("feature", o.detach().clone()))
    res = model(Task(), 1, {'words': s1}, {'words': s2}, None, None, label, weight)
    res['loss'].backward()
    out["feature"] = seen["feature"].numpy()
    out["embs"] = res['embs'].detach().numpy().copy()
    out["logits"] = res['logits'].detach().numpy().copy()
    out["loss"] = np.array(res['loss'].item(), dtype=np.float32)
    for k, p in model.named_parameters():
        out[f"g:{k}"] = p.grad.numpy().copy()
    for kind in ('mse', 'l1', 'focal_mse', 'focal_l1', 'huber'):
        m = build(loss=kind)
        m.train()
        with torch.no_grad():
            r = m(Task(), 1, {'words': s1}, {'words': s2}, None, None, label, weight)
        out[f"loss_{kind}"] = np.array(r['loss'].item(), dtype=np.float32)
    np.savez_compressed(os.path.join(HERE, "stsb_model.npz"), **out)
    print("wrote stsb_model.npz:", {k: v.shape for k, v in out.items() if not k.startswith(("p:", "g:"))})


if __name__ == "__main__":
    main()
