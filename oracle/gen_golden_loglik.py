"""Generate tests/golden/loglik.npz: the reference harness's own loglikelihood answers on two tiny fp32 HF models.

Run:  python -m oracle.gen_golden_loglik          (needs /root/reference; CPU only)

The answers come from the reference's unmodified BaseLM.loglikelihood / _loglikelihood_tokens
(zeroShot/models/models_utils.py) through a stub subclass whose _model_logits_on_dataset is the full HF forward of each
right-padded batch followed by F.log_softmax -- what the reference's per-layer loop computes on such a batch -- and whose
tokenizer maps a string to [ord(c) % V for c in s].  The two models are a Llama with grouped-query attention and a
post-LayerNorm OPT with project_in / project_out and 256 learned positions (room for a shared 64-token page and a
continuation).  The requests include an empty context, contexts longer than max_length (left truncation), requests
repeated verbatim, two splits of one token sequence, and documents of 4 choices sharing a context longer than 64
tokens.  The fixture stores the configs, the weights, the requests, the padded inputs the reference built and its
(logprob, is_greedy) answers; no test reads the reference.
"""
import json
import os
import random
import sys

import numpy as np
import torch
import torch.nn.functional as F

from oracle.gen_golden import OUT, REF

V = 199
EOT = 1
MAX_LENGTH = 200
BATCH = 4
CONFIGS = {
    'llama': dict(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                  num_key_value_heads=2, vocab_size=V, max_position_embeddings=512),
    'opt': dict(hidden_size=64, ffn_dim=128, num_hidden_layers=2, num_attention_heads=4, vocab_size=V,
                max_position_embeddings=256, word_embed_proj_dim=48, do_layer_norm_before=False),
}


def build_model(kind, cfg):
    if kind == 'opt':
        from transformers import OPTConfig, OPTForCausalLM
        return OPTForCausalLM(OPTConfig(**cfg)).float().eval()
    from transformers import LlamaConfig, LlamaForCausalLM
    return LlamaForCausalLM(LlamaConfig(**cfg)).float().eval()


def encode(s):
    return [ord(c) % V for c in s]


def requests(seed=0):
    rnd = random.Random(seed)
    letters = 'abcdefghijklmnopqrstuvwxyz ,.'

    def text(n):
        return ''.join(rnd.choice(letters) for _ in range(n))
    reqs = [('', ' first'), ('', 'x'), ('ab', 'c'), ('a', 'bc')]               # empty contexts; one sequence, two splits
    for _ in range(3):                                                          # multiple choice, shared context > 64
        ctx = text(rnd.randint(70, 150))
        reqs += [(ctx, ' ' + text(rnd.randint(1, 12))) for _ in range(4)]
    reqs += [(text(rnd.randint(210, 260)), ' ' + text(rnd.randint(1, 8))) for _ in range(3)]   # left truncation
    reqs += [(text(rnd.randint(1, 40)), text(rnd.randint(1, 20))) for _ in range(6)]
    reqs += [reqs[5], reqs[9], reqs[-1]]                                        # repeated verbatim
    return reqs


def main():
    sys.path.insert(0, os.path.join(REF, 'zeroShot'))
    from models.models_utils import BaseLM

    class StubLM(BaseLM):
        def __init__(self, model):
            super().__init__()
            self.model, self.inps = model, []

        eot_token_id = property(lambda self: EOT)
        max_length = property(lambda self: MAX_LENGTH)
        max_gen_toks = property(lambda self: 0)
        batch_size = property(lambda self: BATCH)
        device = property(lambda self: 'cpu')

        def tok_encode(self, s):
            return encode(s)

        def tok_decode(self, t):
            raise NotImplementedError

        def _model_generate(self, *a):
            raise NotImplementedError

        def _model_call(self, inps):
            return self.model(inps).logits

        def _model_logits_on_dataset(self, dataset_inps):
            self.inps = [b.clone() for b in dataset_inps]
            with torch.no_grad():
                return [F.log_softmax(self._model_call(b).float(), dim=-1) for b in dataset_inps]

    reqs = requests()
    out = dict(contexts=np.array([c for c, _ in reqs]), continuations=np.array([x for _, x in reqs]),
               meta=np.array(json.dumps(dict(V=V, eot=EOT, max_length=MAX_LENGTH, batch_size=BATCH, configs=CONFIGS))))
    for kind, cfg in CONFIGS.items():
        torch.manual_seed(1)
        model = build_model(kind, cfg)
        lm = StubLM(model)
        ans = lm.loglikelihood(reqs)
        width = max(b.shape[1] for b in lm.inps)
        rows = [np.pad(r.numpy(), (0, width - r.shape[0])) for b in lm.inps for r in b]
        out[f'{kind}_inps'] = np.stack(rows)
        out[f'{kind}_logprob'] = np.array([a[0] for a in ans], dtype=np.float64)
        out[f'{kind}_greedy'] = np.array([a[1] for a in ans], dtype=bool)
        for k, v in model.state_dict().items():
            out[f'{kind}/{k}'] = v.numpy()
    path = os.path.join(OUT, 'loglik.npz')
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
