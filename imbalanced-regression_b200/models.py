"""models.py -- STS-B-DIR's sentence-pair model (sts-b-dir/models.py) on libdirb200.

build_model(args, vocab, pretrained_embs, tasks) builds the reference's MultiTaskModel: a word embedding, a 2-layer
bidirectional LSTM (rnn.LSTM) shared by both sentences, the masked max over time, the pair feature
[u, v, |u - v|, u * v] (fp32 [B, 8 d_hid]), optional FDS (fds_variants.FDSSTSB) and a Linear(8 d_hid, 1) regressor
(dirb200_linear1_fwd / _bwd).  state_dict() keys and shapes are the reference's, AllenNLP module names included.

The AllenNLP 0.5 pieces the reference uses are restated:
* Embedding(V, d_word, padding_index, trainable): a [V, d_word] weight, frozen when GloVe is used without
  --train_words;
* Highway with n_layers_highway = 0 layers is the identity; more layers are refused;
* the 'lstm' seq2seq wrapper runs the LSTM packed by the mask's lengths (rnn.LSTM.forward_padded);
* get_text_field_mask(s) = (ids != 0).

Inputs are token ids, [B, T] int64 or {'words': ids}; mask1 / mask2, when given, are the masks of those ids (the
reference's encoder then expects already-embedded inputs, a path its trainer never takes).  A mask must be a prefix of
ones of length >= 1 per row, as packed sequences assume.

Dropout (training mode, p = args.dropout) is drawn with torch's default generator on the inputs' device, in this
order: s1 embedding [B, T1, d_word], s2 embedding [B, T2, d_word], s1 encoder output [B, T1, 2 d_hid], s2 encoder output
[B, T2, 2 d_hid]; each a bernoulli(1 - p) mask scaled by 1 / (1 - p).  HeadlessPairEncoder.last_dropout keeps the four
multipliers of the last training forward so a test can redraw them.
"""
import logging

import torch
import torch.nn as nn
import torch.nn.functional as F

import _lib
from fds_variants import FDSSTSB
from rnn import LSTM, pad64
from resnet import _Linear1Fn
import loss as _loss


def build_model(args, vocab, pretrained_embs, tasks):
    d_word, n_layers_highway = args.d_word, args.n_layers_highway
    if n_layers_highway > 0:
        raise ValueError(f"--n_layers_highway {n_layers_highway}: highway layers are not built (only 0 is supported)")
    if args.glove:
        word_embs, train_embs = pretrained_embs, bool(args.train_words)
    else:
        logging.info("\tLearning embeddings from scratch!")
        word_embs, train_embs = None, True
    word_embedder = Embedding(vocab.get_vocab_size('tokens'), d_word, weight=word_embs, trainable=train_embs,
                              padding_index=vocab.get_token_index('@@PADDING@@'))
    text_field_embedder = BasicTextFieldEmbedder({"words": word_embedder})
    phrase_layer = _LstmWrapper(LSTM(d_word, args.d_hid, args.n_layers_enc, bidirectional=True, batch_first=True))
    pair_encoder = HeadlessPairEncoder(vocab, text_field_embedder, n_layers_highway, phrase_layer,
                                       dropout=args.dropout)
    d_pair = 2 * args.d_hid
    fds = None
    if args.fds:
        fds = FDSSTSB(feature_dim=d_pair * 4, bucket_num=args.bucket_num, bucket_start=args.bucket_start,
                      start_update=args.start_update, start_smooth=args.start_smooth, kernel=args.fds_kernel,
                      ks=args.fds_ks, sigma=args.fds_sigma, momentum=args.fds_mmt)
    model = MultiTaskModel(args, pair_encoder, fds)
    build_regressor(tasks, model, d_pair)
    if args.cuda >= 0:
        model = model.cuda()
    return model


def build_regressor(tasks, model, d_pair):
    for task in tasks:
        model.build_regressor(task, d_pair * 4)


class Embedding(nn.Module):
    def __init__(self, num_embeddings, embedding_dim, weight=None, trainable=True, padding_index=None):
        super().__init__()
        self.num_embeddings, self.output_dim, self.padding_index = num_embeddings, embedding_dim, padding_index
        if weight is None:
            weight = torch.empty(num_embeddings, embedding_dim)
            nn.init.xavier_uniform_(weight)
        elif tuple(weight.shape) != (num_embeddings, embedding_dim):
            raise ValueError("A weight matrix was passed with contradictory embedding shapes.")
        self.weight = nn.Parameter(weight.detach().clone().float(), requires_grad=trainable)
        if padding_index is not None:      # AllenNLP's Embedding zeroes the padding row, given weights included
            with torch.no_grad():
                self.weight[padding_index].fill_(0)

    def get_output_dim(self):
        return self.output_dim


class BasicTextFieldEmbedder(nn.Module):
    def __init__(self, token_embedders):
        super().__init__()
        self._token_embedders = token_embedders
        for key, emb in token_embedders.items():
            self.add_module(f"token_embedder_{key}", emb)

    def get_output_dim(self):
        return sum(e.get_output_dim() for e in self._token_embedders.values())


class _LstmWrapper(nn.Module):
    """AllenNLP's PytorchSeq2SeqWrapper: holds the LSTM as `_module` (the state_dict prefix)."""

    def __init__(self, module):
        super().__init__()
        self._module = module

    def get_output_dim(self):
        return self._module.get_output_dim()


def _dropout_mult(shape, p, device):
    return torch.empty(shape, device=device).bernoulli_(1 - p).div_(1 - p)


class _EmbedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, weight, ids, lens, dmul, Dp, padding_index):
        M, T = ids.shape
        V, D = weight.shape
        x = torch.empty(T, M, Dp, dtype=torch.bfloat16, device=ids.device)
        _lib.call("dirb200_embed_gather", _lib.ptr(ids), _lib.ptr(lens), _lib.ptr(weight), _lib.ptr(dmul), V, M, T, D,
                  Dp, _lib.ptr(x), _lib.stream_ptr())
        ctx.save_for_backward(ids, lens, dmul)
        ctx.shape = (V, D, Dp)
        ctx.padding_index = -1 if padding_index is None else padding_index
        return x

    @staticmethod
    def backward(ctx, gx):
        if not ctx.needs_input_grad[0]:
            return None, None, None, None, None, None
        ids, lens, dmul = ctx.saved_tensors
        V, D, Dp = ctx.shape
        M, T = ids.shape
        dw = torch.empty(V, D, dtype=torch.float32, device=ids.device)
        _lib.call("dirb200_embed_grad", _lib.ptr(ids), _lib.ptr(lens), _lib.ptr(gx.contiguous()), _lib.ptr(dmul), V,
                  M, T, D, Dp, ctx.padding_index, _lib.ptr(dw), _lib.stream_ptr())
        return dw, None, None, None, None, None


class _PairPoolFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, lens, dmul, B, H, Hp):
        T = y.shape[0]
        feat = torch.empty(B, 8 * H, dtype=torch.float32, device=y.device)
        arg = torch.empty(2 * B, 2 * H, dtype=torch.int32, device=y.device)
        _lib.call("dirb200_pair_maxpool_fwd", _lib.ptr(y), _lib.ptr(lens), _lib.ptr(dmul), B, T, H, Hp,
                  _lib.ptr(feat), _lib.ptr(arg), _lib.stream_ptr())
        # FDS.smooth calibrates the returned feature in place (as sts-b-dir/fds.py:135 does), so u and v are kept
        # from a copy
        ctx.save_for_backward(feat.clone(), arg, dmul)
        ctx.dims = (B, T, H, Hp)
        return feat

    @staticmethod
    def backward(ctx, g):
        feat, arg, dmul = ctx.saved_tensors
        B, T, H, Hp = ctx.dims
        dy = torch.empty(T, 2 * B, 2 * Hp, dtype=torch.bfloat16, device=g.device)
        _lib.call("dirb200_pair_maxpool_bwd", _lib.ptr(g.contiguous()), _lib.ptr(feat), _lib.ptr(arg), _lib.ptr(dmul),
                  B, T, H, Hp, _lib.ptr(dy), _lib.stream_ptr())
        return dy, None, None, None, None, None


def _ids(s):
    return s['words'] if isinstance(s, dict) else s


def _lengths(ids, mask):
    """Row lengths from the mask (default ids != 0); the mask must be a prefix of ones, each row at least 1 long."""
    mask = (ids != 0) if mask is None else mask.bool()
    lens = mask.sum(1)
    T = ids.shape[1]
    if not torch.equal(mask, torch.arange(T, device=ids.device)[None, :] < lens[:, None]):
        raise ValueError("models: every mask row must be a prefix of ones (packed sequences)")
    if int(lens.min()) < 1:
        raise ValueError("models: every sentence needs at least one token (zero-length row)")
    return lens


class HeadlessPairEncoder(nn.Module):
    def __init__(self, vocab, text_field_embedder, num_highway_layers, phrase_layer, dropout=0.2, mask_lstms=True):
        super().__init__()
        if num_highway_layers > 0:
            raise ValueError(f"--n_layers_highway {num_highway_layers}: highway layers are not built")
        if not mask_lstms:
            raise ValueError("HeadlessPairEncoder: only the masked LSTM (mask_lstms=True) is built")
        self._text_field_embedder = text_field_embedder
        self._phrase_layer = phrase_layer
        self.pad_idx = vocab.get_token_index(getattr(vocab, '_padding_token', '@@PADDING@@'))
        self.output_dim = phrase_layer.get_output_dim()
        self.dropout = dropout
        self.last_dropout = None

    def forward(self, s1, s2, m1=None, m2=None):
        ids1, ids2 = _ids(s1), _ids(s2)
        _lib.require_cuda(ids1, ids2)
        B = ids1.shape[0]
        if ids2.shape[0] != B:
            raise ValueError("models: s1 and s2 must have the same batch size")
        lstm = self._phrase_layer._module
        emb = self._text_field_embedder.token_embedder_words
        H, Hp, D = lstm.hidden_size, lstm.hidden_p, emb.output_dim
        T1, T2 = ids1.shape[1], ids2.shape[1]
        T = max(T1, T2)
        lens = torch.cat([_lengths(ids1, m1), _lengths(ids2, m2)]).to(torch.int32)
        ids = torch.cat([F.pad(ids1, (0, T - T1)), F.pad(ids2, (0, T - T2))]).to(torch.int64).contiguous()
        if int(ids.min()) < 0 or int(ids.max()) >= emb.num_embeddings:
            raise ValueError("models: token id outside the vocabulary")
        de = do = None
        if self.training and self.dropout > 0:
            p, dev = self.dropout, ids.device
            m1e, m2e = _dropout_mult((B, T1, D), p, dev), _dropout_mult((B, T2, D), p, dev)
            m1o, m2o = _dropout_mult((B, T1, 2 * H), p, dev), _dropout_mult((B, T2, 2 * H), p, dev)
            self.last_dropout = (m1e, m2e, m1o, m2o)
            de = torch.cat([F.pad(m1e, (0, 0, 0, T - T1)), F.pad(m2e, (0, 0, 0, T - T2))]).contiguous()
            do = torch.cat([F.pad(m1o, (0, 0, 0, T - T1)), F.pad(m2o, (0, 0, 0, T - T2))]).contiguous()
        x = _EmbedFn.apply(emb.weight, ids, lens, de, lstm.input_p, emb.padding_index)
        y = lstm.forward_padded(x, lens)
        return _PairPoolFn.apply(y, lens, do, B, H, Hp)


class MultiTaskModel(nn.Module):
    def __init__(self, args, pair_encoder, FDS=None):
        super().__init__()
        self.args = args
        self.pair_encoder = pair_encoder
        self.FDS = FDS
        self.start_smooth = args.start_smooth

    def build_regressor(self, task, d_inp):
        setattr(self, '%s_pred_layer' % task.name, nn.Linear(d_inp, 1))

    def forward(self, task=None, epoch=None, input1=None, input2=None, mask1=None, mask2=None, label=None,
                weight=None):
        pred_layer = getattr(self, '%s_pred_layer' % task.name)
        pair_emb = self.pair_encoder(input1, input2, mask1, mask2)
        pair_emb_s = pair_emb
        if self.training and self.FDS is not None and epoch >= self.start_smooth:
            pair_emb_s = self.FDS.smooth(pair_emb_s, label, epoch)
        logits = _Linear1Fn.apply(pair_emb_s.contiguous(), pred_layer.weight.view(-1), pred_layer.bias)
        out = {}
        if self.training and self.FDS is not None:
            out['embs'] = pair_emb
            out['labels'] = label
        target = label / 5.
        if self.args.loss == 'huber':
            loss = _loss.weighted_huber_loss(logits, target, weight, beta=self.args.huber_beta)
        elif self.args.loss in ('focal_mse', 'focal_l1'):
            loss = getattr(_loss, f"weighted_{self.args.loss}_loss")(logits, target, weight, beta=20)
        else:
            loss = getattr(_loss, f"weighted_{self.args.loss}_loss")(logits, target, weight)
        out['logits'] = logits
        task.scorer(logits.squeeze(-1).detach().cpu().numpy(), label.squeeze(-1).detach().cpu().numpy())
        out['loss'] = loss
        return out
