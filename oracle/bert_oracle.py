"""Plain-function restatement of BERT's forward as training/stabletts/matcha/onnx/bert-export.py exports it (transformers'
BertModel on one sentence, attention mask all ones, token types 0, returning hidden_states[-3]), in PyTorch CPU ops, in any
float dtype.  `sd` is a BertModel state dict; `bt` the shape (config.bert_config), whose cv_layers layers run."""
import torch
import torch.nn.functional as F


def bert_features(sd, bt, ids, dtype=torch.float64):
    """ids: the word-piece ids of one sentence.  Returns the output of layer cv_layers [L, hidden]."""
    w = lambda k: torch.as_tensor(sd[k]).to(dtype)
    ids = torch.as_tensor(ids, dtype=torch.long).reshape(-1)
    L, H, nh, eps = ids.numel(), bt["cv_hidden"], bt["cv_heads"], bt["cv_ln_eps"]
    ln = lambda t, p: F.layer_norm(t, t.shape[-1:], w(p + ".weight"), w(p + ".bias"), eps=eps)
    e = "embeddings."
    x = w(e + "word_embeddings.weight")[ids] + w(e + "token_type_embeddings.weight")[0]
    x = ln(x + w(e + "position_embeddings.weight")[:L], e + "LayerNorm")
    dk = H // nh
    for l in range(bt["cv_layers"]):
        pre = "encoder.layer.%d." % l
        lin = lambda t, n: t @ w(pre + n + ".weight").T + w(pre + n + ".bias")
        q = lin(x, "attention.self.query").reshape(L, nh, dk).transpose(0, 1)
        k = lin(x, "attention.self.key").reshape(L, nh, dk).transpose(0, 1)
        v = lin(x, "attention.self.value").reshape(L, nh, dk).transpose(0, 1)
        a = torch.softmax(q @ k.transpose(1, 2) / dk ** 0.5, dim=-1) @ v
        x = ln(x + lin(a.transpose(0, 1).reshape(L, H), "attention.output.dense"), pre + "attention.output.LayerNorm")
        h = F.gelu(lin(x, "intermediate.dense"))
        x = ln(x + lin(h, "output.dense"), pre + "output.LayerNorm")
    return x


def flops(bt, L):
    """Multiply-adds x 2 of one sentence of L word pieces: the layers' GEMMs and the attention's two products."""
    H, Fh = bt["cv_hidden"], bt["cv_ffn"]
    return bt["cv_layers"] * (2.0 * L * (4 * H * H + 2 * H * Fh) + 4.0 * L * L * H)
