"""Adapter from the reference's zero-shot harness (zeroShot/evaluator.py) to a packed model.

The harness's tasks ask an `LM` for `loglikelihood(requests)`: for each (context, continuation) string pair, the sum of
the continuation tokens' log-probabilities and whether greedy decoding would produce the continuation.  `PackedLM`
answers it with quip_b200.decode.score -- chunked prefill straight into the KV cache, lm_head at the scored positions
only and the log-softmax of csrc/logprob.cu -- on the model as it is (packed QuantLinear layers included):

    lm = PackedLM(model, tokenizer, batch_size=32, max_length=2048)
    results = evaluator.evaluate(lm=lm, task_dict=tasks.get_task_dict(['arc_easy', 'lambada', 'piqa', 'storycloze']))

The other request types of the harness (loglikelihood_rolling, greedy_until) are not used by those tasks and raise.
"""
from . import decode


class PackedLM:
    """The reference harness's LM.loglikelihood contract on strings for a packed Llama or OPT model.

    tokenizer: anything with encode(s, add_special_tokens=False) -> ids and eos_token_id (the end-of-text id the
    harness substitutes for an empty context).  batch_size, max_length: as the harness's BaseLM has them (requests per
    batch; the input window, left-truncated).  score_kw: further arguments of decode.score (kv_dtype,
    prefill_chunk_size, share_prompt_prefixes)."""

    def __init__(self, model, tokenizer, batch_size, max_length, **score_kw):
        self.model, self.tokenizer = model, tokenizer
        self.batch_size, self.max_length = int(batch_size), int(max_length)
        self.score_kw = score_kw

    @property
    def eot_token_id(self):
        return self.tokenizer.eos_token_id

    def tok_encode(self, string):
        return self.tokenizer.encode(string, add_special_tokens=False)

    def loglikelihood(self, requests):
        """requests: (context, continuation) string pairs -> [(logprob, is_greedy)] in the same order."""
        ctxs, conts = [], []
        for context, continuation in requests:
            ctxs.append([self.eot_token_id] if context == '' else self.tok_encode(context))
            conts.append(self.tok_encode(continuation))
        if not ctxs:
            return []
        return decode.score(self.model, ctxs, conts, batch_size=self.batch_size, max_length=self.max_length,
                            **self.score_kw)

    def loglikelihood_rolling(self, requests):
        raise NotImplementedError('PackedLM answers loglikelihood requests only (the ArcE, LAMBADA, PiQA and '
                                  'StoryCloze tasks use nothing else)')

    def greedy_until(self, requests):
        raise NotImplementedError('PackedLM answers loglikelihood requests only (the ArcE, LAMBADA, PiQA and '
                                  'StoryCloze tasks use nothing else)')
