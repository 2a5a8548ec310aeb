"""STS-B-DIR's sentence-pair model at the reference's defaults (batch 128, T = 40, d_word 300, d_hid 1500, 2 layers,
seeded synthetic lengths): the native training step (forward, backward, optim.Adam after clip_grad_norm_(5)), eval
forward at batch 128 and 1, and the recurrent step kernels alone with the FLOPs / bytes each needs, against
oracle/stsb_ref-style torch on cuDNN's packed LSTM in fp32 (TF32 off and on).  Prints one JSON line with the card name
and power limit read in the same run, and peak memory.

    python tools/stsb_model_bench.py [--steps 10] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "imbalanced-regression_b200")]

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


class Vocab:
    def get_vocab_size(self, ns):
        return 20000

    def get_token_index(self, tok):
        return 0


class Task:
    name = 'sts-b'

    def scorer(self, logits, labels):
        pass


def batch(B, T, V, dev, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(2):
        L = torch.randint(5, T + 1, (B,), generator=g)
        L[0] = T
        ids = torch.randint(1, V, (B, T), generator=g) * (torch.arange(T)[None] < L[:, None])
        out.append(ids.to(dev))
    return out[0], out[1], (torch.rand(B, 1, generator=g) * 5).to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import _lib
    import optim
    from models import build_model
    dev = torch.device("cuda", 0)
    B, T, D, H, V = 128, 40, 300, 1500, 20000
    args = SimpleNamespace(d_word=D, n_layers_highway=0, glove=1, train_words=0, d_hid=H, n_layers_enc=2, dropout=0.2,
                           fds=0, start_smooth=1, cuda=0, loss='mse', huber_beta=0.5)
    torch.manual_seed(0)
    model = build_model(args, Vocab(), torch.randn(V, D), [Task()])
    s1, s2, label = batch(B, T, V, dev, 0)
    params = [p for p in model.parameters() if p.requires_grad]
    opt = optim.Adam(params, lr=1e-4)
    res = {"card": card(), "batch": B, "T": T, "d_word": D, "d_hid": H}

    def train_step():
        model.train()
        out = model(Task(), 0, s1, s2, label=label)
        opt.zero_grad()
        out['loss'].backward()
        torch.nn.utils.clip_grad_norm_(params, 5.0)
        opt.step()

    torch.cuda.reset_peak_memory_stats()
    res["native_train_step_ms"] = timed(train_step, a.steps, a.warmup)
    res["native_train_peak_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
    model.eval()
    with torch.no_grad():
        res["native_eval_b128_ms"] = timed(lambda: model.pair_encoder(s1, s2), a.steps, a.warmup)
        res["native_eval_b1_ms"] = timed(lambda: model.pair_encoder(s1[:1], s2[:1]), a.steps, a.warmup)

    # the recurrent step kernels alone, at M = 2B, Hp = 1536
    lstm = model.pair_encoder._phrase_layer._module
    M, Hp = 2 * B, lstm.hidden_p
    lens = torch.full((M,), T, dtype=torch.int32, device=dev)
    xproj = torch.zeros(T, M, 8 * Hp, dtype=torch.bfloat16, device=dev)
    whh = torch.zeros(2, 4 * Hp, Hp, dtype=torch.bfloat16, device=dev)
    bias = torch.zeros(2, 4 * Hp, device=dev)
    h = torch.zeros(2, T + 1, M, Hp, dtype=torch.bfloat16, device=dev)
    c = torch.zeros(2, T + 1, M, Hp, device=dev)
    gates = torch.zeros(2, T, M, 4 * Hp, device=dev)
    y = torch.zeros(T, M, 2 * Hp, dtype=torch.bfloat16, device=dev)
    fwd = lambda: _lib.call("dirb200_lstm_fwd_step", _lib.ptr(xproj), _lib.ptr(whh), _lib.ptr(bias), _lib.ptr(lens),
                            T, M, Hp, 1, 5, _lib.ptr(h), _lib.ptr(c), _lib.ptr(gates), _lib.ptr(y), _lib.stream_ptr())
    dg = torch.zeros(2, T, M, 4 * Hp, dtype=torch.bfloat16, device=dev)
    dgt = torch.zeros(T, M, 8 * Hp, dtype=torch.bfloat16, device=dev)
    dc = torch.zeros(2, 2, M, Hp, device=dev)
    bwd = lambda: _lib.call("dirb200_lstm_bwd_step", _lib.ptr(whh), _lib.ptr(y), _lib.ptr(gates), _lib.ptr(c),
                            _lib.ptr(lens), T, M, Hp, 5, _lib.ptr(dc), _lib.ptr(dg), _lib.ptr(dgt), _lib.stream_ptr())
    flop = 2 * 2 * M * 4 * Hp * Hp                       # both directions
    fwd_bytes = 2 * (4 * Hp * Hp * 2 + M * Hp * 2 + M * 4 * Hp * 2 + M * Hp * 4 * 2 + M * 4 * Hp * 4 + 2 * M * Hp * 2)
    bwd_bytes = 2 * (4 * Hp * Hp * 2 + M * 4 * Hp * 2 + M * Hp * 2 + M * 4 * Hp * 4 + 2 * M * Hp * 4 + 2 * M * Hp * 4
                     + 2 * M * 4 * Hp * 2)
    for name, fn, by in (("fwd_step", fwd, fwd_bytes), ("bwd_step", bwd, bwd_bytes)):
        ms = timed(fn, 200, 20)
        res[f"{name}_us"] = ms * 1e3
        res[f"{name}_tflops"] = flop / (ms * 1e-3) / 1e12
        res[f"{name}_gbytes"] = by / 1e9
        res[f"{name}_tb_per_s"] = by / (ms * 1e-3) / 1e12

    # comparison arm: torch's packed cuDNN LSTM in fp32 with the same embedding / max-pool / regressor in torch
    ref = torch.nn.LSTM(D, H, 2, bidirectional=True, batch_first=True).to(dev)
    ref.load_state_dict(lstm.state_dict())
    emb = model.pair_encoder._text_field_embedder.token_embedder_words.weight
    lin = torch.nn.Linear(8 * H, 1).to(dev)
    ropt = torch.optim.Adam([p for p in ref.parameters()] + list(lin.parameters()), lr=1e-4)
    drop = torch.nn.Dropout(0.2)

    def enc(s):
        L = (s != 0).sum(1)
        pk = torch.nn.utils.rnn.pack_padded_sequence(drop(emb[s]), L.cpu(), batch_first=True, enforce_sorted=False)
        o, _ = ref(pk)
        o, _ = torch.nn.utils.rnn.pad_packed_sequence(o, batch_first=True, total_length=s.shape[1])
        o = drop(o).masked_fill(~(torch.arange(s.shape[1], device=dev)[None] < L[:, None])[..., None], float("-inf"))
        return o.max(1).values

    def ref_step():
        u, v = enc(s1), enc(s2)
        loss = ((lin(torch.cat([u, v, (u - v).abs(), u * v], 1)) - label / 5) ** 2).mean()
        ropt.zero_grad()
        loss.backward()
        torch.nn.utils.clip_grad_norm_(list(ref.parameters()) + list(lin.parameters()), 5.0)
        ropt.step()

    for tf32 in (False, True):
        torch.backends.cuda.matmul.allow_tf32 = tf32
        torch.backends.cudnn.allow_tf32 = tf32
        tag = "tf32" if tf32 else "fp32"
        torch.cuda.reset_peak_memory_stats()
        ref.train()
        drop.train()
        res[f"cudnn_{tag}_train_step_ms"] = timed(ref_step, a.steps, a.warmup)
        res[f"cudnn_{tag}_train_peak_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
        ref.eval()
        drop.eval()
        with torch.no_grad():
            res[f"cudnn_{tag}_eval_b128_ms"] = timed(lambda: (enc(s1), enc(s2)), a.steps, a.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
