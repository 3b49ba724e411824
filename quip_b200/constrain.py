"""Token automata for constrained generation (generate(..., token_constraint=...)).

A TokenAutomaton is a finite set of states; each state allows a non-empty set of token ids and maps each of them to
a next state.  generate() keeps one current state per row on the device, masks the row's logits to the allowed ids
of its state (quip_constrain_mask) and moves the state over each committed token (quip_constrain_advance), inside the
captured decode step.  A token the state has no transition for leaves the state unchanged; that happens only when no
allowed entry of the masked row was finite (for example min_new_tokens banning an EOS-only state).

pack_automata turns automata into the device table of include/quip_b200.h: offsets (S + 1), ids and next (nnz) int32,
each automaton's states a disjoint range.
"""
import torch


class TokenAutomaton:
    """A token automaton from explicit transitions {state: {token: next_state}} (states any hashable values, tokens
    ints >= 0) and a start state.  Every state needs at least one allowed token (HF refuses an empty allowed list), and
    every next state must be a state of the automaton.  Token ids are checked against the vocabulary when generate()
    packs the automaton."""

    def __init__(self, transitions, start):
        if not isinstance(transitions, dict) or not transitions:
            raise ValueError('transitions must be a non-empty dict {state: {token: next_state}}')
        self.states = list(transitions)
        index = {s: j for j, s in enumerate(self.states)}
        if start not in index:
            raise ValueError(f'start state {start!r} is not a state of the automaton')
        self.arcs = []                                        # per state index: sorted [(token, next index)]
        for s in self.states:
            arcs = transitions[s]
            if not isinstance(arcs, dict) or not arcs:
                raise ValueError(f'state {s!r} allows no token: every state needs at least one')
            row = []
            for v, nxt in arcs.items():
                if isinstance(v, bool) or not isinstance(v, int) or v < 0:
                    raise ValueError(f'state {s!r}: token ids must be integers >= 0, got {v!r}')
                if nxt not in index:
                    raise ValueError(f'state {s!r}: token {v} leads to {nxt!r}, which is not a state')
                row.append((v, index[nxt]))
            self.arcs.append(sorted(row))
        self._next = [dict(arcs) for arcs in self.arcs]
        self._index = index
        self.start = start

    def allowed(self, state):
        """The sorted token ids `state` allows."""
        return [v for v, _ in self.arcs[self._index[state]]]

    def walk(self, state, tokens):
        """The state reached from `state` over `tokens`; a token without a transition leaves the state unchanged."""
        j = self._index[state]
        for v in tokens:
            j = self._next[j].get(int(v), j)
        return self.states[j]

    @classmethod
    def from_sequences(cls, seqs, eos):
        """The trie that accepts exactly one of the id sequences `seqs` followed by an EOS id (eos: an id or a list of
        ids), then an EOS-only sink: a label set or a multiple choice."""
        eos = [int(eos)] if isinstance(eos, int) else [int(e) for e in eos]
        if not eos or not seqs:
            raise ValueError('from_sequences needs at least one sequence and one EOS id')
        trans, sink = {0: {}}, 'sink'
        for seq in seqs:
            node = 0
            for v in (seq.tolist() if torch.is_tensor(seq) else seq):
                if int(v) in eos:
                    raise ValueError(f'sequence {seq!r} holds an EOS id')
                nxt = trans[node].get(int(v))
                if nxt is None:
                    nxt = len(trans) - (sink in trans)
                    trans[node][int(v)] = nxt
                    trans[nxt] = {}
                node = nxt
            trans[node].update({e: sink for e in eos})
            trans[sink] = {e: sink for e in eos}
        return cls(trans, 0)

    def hf_prefix_allowed_tokens_fn(self, prompt_len):
        """HF's prefix_allowed_tokens_fn(batch_id, input_ids) equivalent of this automaton for a prompt of prompt_len
        tokens: the ids allowed in the state walked from the start over input_ids[prompt_len:]."""
        return lambda batch_id, input_ids: self.allowed(self.walk(self.start, input_ids[prompt_len:].tolist()))


def pack_automata(automata, vocab):
    """The device table of a list of TokenAutomaton or None entries: (offsets (S + 1,), ids (nnz,), next (nnz,)) int32
    CPU tensors and each entry's start state in the table (-1 for None).  An automaton given several times is packed
    once.  Raises ValueError for a token id outside [0, vocab) or an entry that is not an automaton."""
    offsets, ids, nxt, base, starts = [0], [], [], {}, []
    for a in automata:
        if a is None:
            starts.append(-1)
            continue
        if not isinstance(a, TokenAutomaton):
            raise ValueError(f'token_constraint entries must be TokenAutomaton or None, got {type(a).__name__}')
        if id(a) not in base:
            base[id(a)] = b = len(offsets) - 1
            for arcs in a.arcs:
                for v, j in arcs:
                    if v >= vocab:
                        raise ValueError(f'token id {v} of a token automaton lies outside the vocabulary [0, {vocab})')
                    ids.append(v)
                    nxt.append(b + j)
                offsets.append(len(ids))
        starts.append(base[id(a)] + a._index[a.start])
    if len(offsets) > 2 ** 31 - 1 or len(ids) > 2 ** 31 - 1:
        raise ValueError('the packed token automata exceed 2^31 - 1 states or transitions')
    t = lambda x: torch.tensor(x, dtype=torch.int32)
    return t(offsets), t(ids), t(nxt), starts
