"""GPT-3 (1.3B / 2.7B Megatron-style) decoder of mPLUG-Video on the H100 kernels.

Mirrors the reference module `models/modeling_distributed_gpt3.py`: GPT3Config (:459-547),
BatchEncoding (:139-178), DistributedGPT3Tokenizer (:180-319), DistributedGPT3 (:1522-1618).
No megatron_util: tensor-model-parallel size must be 1 (SURVEY.md D6) - the path is pure data
parallel.  Parameter names equal the reference's (`dist_model.language_model....`), including the
per-head [q|k|v] row grouping of query_key_value, so `model/mp_rank_00_model_states.pt` loads as is.

Host-side API helpers whose behaviour has to match the reference token for token - BatchEncoding (:139-176), the
top-k / top-p logit filters and `sample` (:1369-1443), BeamHypotheses (:1908-1961) - keep the reference's control flow
and messages on purpose (they are thin re-statements of upstream Megatron / HF utilities and are pinned against the
reference's own outputs in tests/golden/tiny_generate.pt); everything that touches the device - parameter containers,
the KV cache, the decoding loops run_sample / run_beam_search, the captured single-token step - is this package's own.
"""
import json
import math
import os
import os.path as osp

import numpy as np
import torch
import torch.nn as nn

from ymp import functional as YF

from ._params import EmbedHolder, Holder, add_param, named_param_list


class AttrDict(dict):
    """addict.Dict-like result container (attribute access; missing keys -> None)."""
    __getattr__ = dict.get
    __setattr__ = dict.__setitem__


class GPT3Config:
    model_type = 'gpt3'

    def __init__(self, vocab_size=25600, hidden_size=768, ffn_hidden_size=None, num_hidden_layers=12,
                 num_attention_heads=12, intermediate_size=3072, hidden_act='gelu', hidden_dropout_prob=0.1,
                 attention_probs_dropout_prob=0.1, max_position_embeddings=2048, type_vocab_size=2,
                 layernorm_epsilon=1e-12, bias_gelu_fusion=True, fp32_residual_connection=False,
                 sequence_parallel=False, fp16=False, bf16=False, apply_query_key_layer_scaling=True,
                 attention_softmax_in_fp32=False, kv_channels=None, masked_softmax_fusion=True,
                 attention_dropout=0.1, bias_dropout_fusion=True,
                 apply_residual_connection_post_layernorm=False, hidden_dropout=0.1, init_method_std=0.02,
                 eod_id=7, tokens_to_generate=100, top_k=0, top_p=0.9, **kwargs):
        self.vocab_size = vocab_size
        self.hidden_size = hidden_size
        self.ffn_hidden_size = 4 * hidden_size if ffn_hidden_size is None else ffn_hidden_size
        self.num_hidden_layers = num_hidden_layers
        self.num_attention_heads = num_attention_heads
        self.intermediate_size = intermediate_size
        self.hidden_act = hidden_act
        self.hidden_dropout_prob = hidden_dropout_prob
        self.attention_probs_dropout_prob = attention_probs_dropout_prob
        self.max_position_embeddings = max_position_embeddings
        self.type_vocab_size = type_vocab_size
        self.layernorm_epsilon = layernorm_epsilon
        self.layer_norm_eps = layernorm_epsilon
        self.fp16, self.bf16 = fp16, bf16
        assert not (fp16 and bf16)
        assert hidden_size % num_attention_heads == 0
        self.kv_channels = hidden_size // num_attention_heads if kv_channels is None else kv_channels
        self.attention_dropout = attention_dropout
        self.hidden_dropout = hidden_dropout
        self.init_method_std = init_method_std
        self.apply_query_key_layer_scaling = apply_query_key_layer_scaling
        self.apply_residual_connection_post_layernorm = apply_residual_connection_post_layernorm
        self.sequence_parallel = sequence_parallel
        self.eod_id, self.tokens_to_generate, self.top_k, self.top_p = eod_id, tokens_to_generate, top_k, top_p
        self.checkpoint_activations = False   # set from megatron_cfg by DistributedGPT3
        for k, v in kwargs.items():
            setattr(self, k, v)
        if apply_residual_connection_post_layernorm or sequence_parallel or fp32_residual_connection:
            raise NotImplementedError("unsupported GPT3Config option for the H100 path")

    @classmethod
    def from_json_file(cls, path):
        with open(path, 'r') as f:
            return cls(**json.load(f))

    @classmethod
    def from_pretrained(cls, model_dir):
        return cls.from_json_file(osp.join(model_dir, 'config.json'))

    def to_dict(self):
        return dict(self.__dict__)

    def engine_cfg(self, training=False):
        """Dims + the dropout setting of one decoder pass: hidden_dropout / attention_dropout are live only in
        train() mode (the reference keeps the frozen decoder in train mode during training).  checkpoint_activations:
        a pass that needs a backward recomputes each layer's activations there instead of keeping them."""
        return dict(vocab_size=self.vocab_size, hidden_size=self.hidden_size, ffn_hidden_size=self.ffn_hidden_size,
                    num_hidden_layers=self.num_hidden_layers, num_attention_heads=self.num_attention_heads,
                    max_position_embeddings=self.max_position_embeddings, layernorm_epsilon=self.layernorm_epsilon,
                    hidden_dropout=self.hidden_dropout, attention_dropout=self.attention_dropout, training=bool(training),
                    checkpoint_activations=bool(self.checkpoint_activations))


# ------------------------------------------------------------------------------------------ tokenizer
class JiebaBPETokenizer:
    """BPE tokenizer (tokenizers json) with jieba pre-segmentation, <sep> as BOS and
    <|endoftext|> as EOS/PAD (reference :42-137)."""

    def __init__(self, tokenizer_json_file):
        from tokenizers import Tokenizer
        self.tokenizer = Tokenizer.from_file(tokenizer_json_file)
        try:
            import jieba
            self._cut = lambda s: list(jieba.cut(s))
        except ImportError:  # not in this image: whitespace segmentation keeps the API usable
            self._cut = lambda s: s.split()
        self.eod_id = self.eos_id = self.pad_id = self.tokenizer.token_to_id('<|endoftext|>')
        self.bos_id = self.sep_token = self.tokenizer.token_to_id('<sep>')

    @property
    def vocab_size(self):
        return self.tokenizer.get_vocab_size(with_added_tokens=True)

    @property
    def vocab(self):
        return self.tokenizer.get_vocab(with_added_tokens=True)

    def _ids(self, text, is_code):
        if is_code:
            return self.tokenizer.encode(text, is_pretokenized=False, add_special_tokens=True).ids
        return self.tokenizer.encode(self._cut(text), is_pretokenized=True, add_special_tokens=True).ids

    def tokenize(self, text, is_code=False, add_special_tokens=True):
        ids = self._ids(text, is_code)
        return [self.bos_id] + ids + [self.eos_id] if add_special_tokens else ids

    def tokenize_prompt(self, prompt_text, text, is_code=False, add_special_tokens=True):
        return [[self.bos_id], self._ids(prompt_text, is_code), self._ids(text, is_code), [self.eos_id]]

    def detokenize(self, token_ids):
        return self.tokenizer.decode(token_ids, skip_special_tokens=True)

    eod = property(lambda self: self.eod_id)
    eos = property(lambda self: self.eos_id)
    bos = property(lambda self: self.bos_id)
    pad = property(lambda self: self.pad_id)


class BatchEncoding:
    def __init__(self, data):
        self.data = data

    def __getitem__(self, item):
        if isinstance(item, str):
            return self.data[item]
        raise KeyError("integer indexing is not available for this tokenizer")

    def __getattr__(self, item):
        try:
            return self.__dict__["data"][item]
        except KeyError:
            raise AttributeError(item)

    def __getstate__(self):
        return {"data": self.data}

    def __setstate__(self, state):
        self.__dict__["data"] = state["data"]

    def __repr__(self):
        return str(self.data)

    def keys(self):
        return self.data.keys()

    def values(self):
        return self.data.values()

    def items(self):
        return self.data.items()

    def to(self, device):
        self.data = {k: v.to(device=device) for k, v in self.data.items()}
        return self


class DistributedGPT3Tokenizer:
    def __init__(self, model_dir, sequence_length=128):
        self.tokenizer = JiebaBPETokenizer(osp.join(model_dir, 'tokenizer.json'))
        self.max_length = sequence_length

    def decode(self, tokens, **kwargs):
        if isinstance(tokens, torch.Tensor):
            tokens = tokens.detach().cpu().tolist()
        return self.tokenizer.detokenize(tokens)

    def _fit(self, ids, length):
        """pad with the pad id / cut to `length`; returns (array, number of real tokens)."""
        ids = list(ids)[:length]
        n = len(ids)
        return np.asarray(ids + [self.tokenizer.pad] * (length - n), dtype=np.int64), n

    def _fit_prompt(self, parts, length):
        bos, prompt, text, eos = parts
        if len(bos) + len(prompt) + len(text) + len(eos) > length:
            room = length - len(text) - 2
            if room >= 0 and len(prompt) >= room:   # shorten the prompt first
                prompt = prompt[:room]
            else:                                    # otherwise cut the target
                text = text[:length - 2 - len(prompt)]
        arr, n = self._fit(bos + prompt + text + eos, length)
        return arr, len(prompt), n

    def __call__(self, data, padding='longest', truncation=True, max_length=None, return_tensors='pt',
                 add_special_tokens=True, **kwargs):
        max_length = self.max_length if max_length is None else max_length
        pairs = not isinstance(data[0], str)
        if pairs:
            toks = [self.tokenizer.tokenize_prompt(p, t) for p, t in data]
            longest = max(sum(len(x) for x in t) for t in toks)
            # the reference pads pair inputs to max_length whenever truncation is on (:289-296)
            length = max_length if (truncation or padding == 'max_length') else longest
        else:
            # NB: the reference passes add_special_tokens positionally into `is_code` (:240);
            # keep the observable behaviour: text path, specials always added.
            toks = [self.tokenizer.tokenize(t) for t in data]
            longest = max(len(t) for t in toks)
            if padding == 'max_length':
                length = max_length
            else:
                length = min(longest, max_length) if truncation else longest
        ids, mask, plen = [], [], []
        for t in toks:
            if pairs:
                arr, pl, n = self._fit_prompt(t, length)
                plen.append(pl)
            else:
                arr, n = self._fit(t, length)
            m = np.zeros(length, dtype=np.int64)
            m[:n] = 1
            ids.append(arr)
            mask.append(m)
        out = dict(input_ids=np.stack(ids), attention_mask=np.stack(mask))
        if pairs:
            out["prompt_lengths"] = np.asarray(plen, dtype=np.int64)
        if return_tensors == 'pt':
            out = {k: torch.from_numpy(v).long() for k, v in out.items()}
        return BatchEncoding(out)


# ------------------------------------------------------------------------------------------ model
def _ckpt_name(mp_rank, load_dir, tag):
    return osp.join(load_dir, str(tag), 'mp_rank_{:02d}_model_states.pt'.format(mp_rank))


def pre_load(mp_rank, load_dir, tag=''):
    """{text_decoder}/model/mp_rank_00_model_states.pt['module'] (reference :431-441)."""
    ckpt = torch.load(_ckpt_name(mp_rank, load_dir, tag), map_location='cpu', weights_only=False)
    return ckpt['module']


def _check_tp1(megatron_cfg):
    if not megatron_cfg:
        return
    for k in ('tensor_model_parallel_size', 'model_parallel_size'):
        v = megatron_cfg.get(k, 1)
        if v not in (None, 1):
            raise ValueError(f"megatron_cfg.{k}={v}: the H100 path is pure data parallel; set it to 1 "
                             "(as the reference's own scripts/*.sh:13-14 and retrieval yaml do)")


# ----------------------------------------------------------------------------------------------
# Generation (SURVEY.md 8f N2): the host logic of models/modeling_distributed_gpt3.py:1369-1473,1620-1886,
# 1908-1961 on top of the KV-cache decode path of ymp.engine.
# ----------------------------------------------------------------------------------------------
def modify_logits_for_top_k_filtering(logits, top_k):
    """In place: everything below the k-th largest logit of its row becomes -inf (:1369-1373)."""
    kth = torch.topk(logits, top_k)[0][..., -1, None]
    logits.masked_fill_(logits < kth, float('-Inf'))


def modify_logits_for_top_p_filtering(logits, top_p):
    """In place nucleus filter (:1376-1395): sorted cumulative probability > top_p is dropped, shifted by
    one position so that the token crossing the threshold is kept; the best token always survives."""
    sorted_logits, sorted_indices = torch.sort(logits, descending=True)
    drop = sorted_logits.softmax(dim=-1).cumsum(dim=-1) > top_p
    drop[:, 1:] = drop[:, :-1].clone()
    drop[..., 0] = 0
    logits.masked_fill_(drop.scatter(1, sorted_indices, drop), float('-Inf'))


def sample(logits, top_k=0, top_p=0.0, temperature=1.0, vocab_size=None):
    """One token per row of logits [b, v] (:1398-1446): argmax when top_k == 1, otherwise temperature,
    top-k or top-p filtering and a multinomial draw; clamped into [0, vocab_size)."""
    assert logits.ndim == 2, 'expected the logits to be of [b, v] shape.'
    if top_k == 1:
        assert top_p == 0.0, 'cannot set both greedy and top-p samplings.'
        samples = torch.argmax(logits, dim=-1)
    else:
        logits = logits.clone()
        if temperature != 1.0:
            logits.div_(temperature)
        if top_k > 1:
            assert top_p == 0.0, 'cannot set both top-k and top-p samplings.'
            assert top_k <= logits.size(1), 'top-k is larger than logit size.'
            if vocab_size:
                assert top_k < vocab_size, 'top-k is larger than vocab size.'
            modify_logits_for_top_k_filtering(logits, top_k)
        elif top_p > 0.0:
            assert top_p <= 1.0, 'top-p should be in (0, 1].'
            modify_logits_for_top_p_filtering(logits, top_p)
        samples = torch.multinomial(logits.softmax(dim=-1), num_samples=1).view(-1)
    if vocab_size:
        samples = torch.clamp(samples, min=0, max=(vocab_size - 1))
    return samples


class InferenceParams:
    """Incremental-decoding state (:1449-1473).  The key/value memory of every layer lives in one
    ymp.engine.KVCache (packed QKV rows the attention kernels read in place); `key_value_memory_dict`
    exposes it per layer number for code that only checks for emptiness."""

    def __init__(self, max_batch_size, max_sequence_len):
        self.max_sequence_len = max_sequence_len
        self.max_batch_size = max_batch_size
        self.sequence_len_offset = 0
        self.batch_size_offset = 0
        self.key_value_memory_dict = {}
        self.cache = None
        self.token_step = None   # ymp.engine.TokenStep once this call's single-token steps have been validated
        # batched beam search: single-token steps of up to ops.SKINNY_WIDE_MAX_ROWS rows run the captured skinny step
        # (otherwise rows beyond ops.SKINNY_MAX_ROWS take the tensor-core path), and the first call fills cache slot
        # b * prefill_stride from input row b
        self.wide_step = False
        self.prefill_stride = 1

    def swap_key_value_dict(self, batch_idx):
        'swap between batches'
        if self.cache is None:
            raise ValueError('should not swap when dict in empty')
        assert len(batch_idx) == self.cache.B  # make sure batch size is the same
        self.cache.reorder(torch.as_tensor(batch_idx, device=self.cache.qkv[0].device, dtype=torch.long))
        self.key_value_memory_dict = {i + 1: t for i, t in enumerate(self.cache.qkv)}


class BeamHypotheses:
    """n-best list of finished hypotheses (:1908-1961).  score = sum_logprobs / len(hyp) ** length_penalty,
    where hyp is the (padded) token row handed in by beam_search."""

    def __init__(self, num_beams, length_penalty=1.0, early_stopping=False):
        self.length_penalty = length_penalty
        self.early_stopping = early_stopping
        self.num_beams = num_beams
        self.beams = []
        self.worst_score = 1e9

    def __len__(self):
        return len(self.beams)

    def add(self, hyp, sum_logprobs, beam_indices=None):
        score = sum_logprobs / (hyp.shape[-1] ** self.length_penalty)
        if len(self) < self.num_beams or score > self.worst_score:
            self.beams.append((score, hyp, beam_indices))
            if len(self) > self.num_beams:
                ranked = sorted((s, idx) for idx, (s, _, _) in enumerate(self.beams))
                del self.beams[ranked[0][1]]
                self.worst_score = ranked[1][0]
            else:
                self.worst_score = min(score, self.worst_score)

    def is_done(self, best_sum_logprobs, cur_len):
        if len(self) < self.num_beams:
            return False
        if self.early_stopping:
            return True
        return self.worst_score >= best_sum_logprobs / cur_len ** self.length_penalty


def run_sample(step, tokens, lengths, n_query, *, tokens_to_generate, eod_id, max_position_embeddings, top_k, top_p,
               temperature=1.0, vocab_size=None, termination_id=None, use_eod_token_for_early_termination=True,
               stop_on_double_eol=False, stop_on_eol=False):
    """DistributedGPT3.sample's loop (:1620-1741) over a decode callback.
    step(new_tokens [B, n], first) -> next-token logits [B, V] of the last position (fp32); the callback owns
    the KV cache and the visual prefix (n_query positions, fed on the first call)."""
    B = tokens.size(0)
    dev = tokens.device
    lengths = lengths.to(dev)
    tokens = torch.cat((tokens, torch.full((B, tokens_to_generate), eod_id, dtype=torch.long, device=dev)), dim=-1)
    max_len = min(tokens.size(1), max_position_embeddings)
    min_prompt = int(lengths.min().item())
    if min_prompt >= max_len:
        raise ValueError('context length + tokens_to_generate too large')
    if termination_id is None:
        termination_id = eod_id
    finished = torch.zeros(B, dtype=torch.bool, device=dev)
    prev = 0
    ctx = min_prompt
    for ctx in range(min_prompt, max_len):
        logits = step(tokens[:, prev:ctx], ctx == min_prompt)
        new = sample(logits, top_k=top_k, top_p=top_p, temperature=temperature, vocab_size=vocab_size)
        started = lengths <= ctx  # samples whose prompt has been consumed start writing their own tokens
        tokens[started, ctx] = new[started]
        prev = ctx
        if stop_on_double_eol:
            hit = ((new == 628) | ((new == 198) & (tokens[:, ctx - 1] == 198))) & started
        elif stop_on_eol:
            hit = ((new == 628) | (new == 198)) & started
        else:
            hit = (new == termination_id) & started
        finished |= hit
        if use_eod_token_for_early_termination and bool(finished.all()):
            break
    # the reference slices with the context length that still counts the prefix positions (:1740)
    return tokens[:, :ctx + n_query + 1]


def _prefill_runs(groups, plens):
    """Refills of one step that can share a prefill launch: groups whose clips have one prompt length and whose slots
    are equally spaced.  groups ascending; returns [(prompt_length, first_group, group_stride, [groups])]."""
    by_len = {}
    for g, p in zip(groups, plens):
        by_len.setdefault(int(p), []).append(g)
    runs = []
    for p, gs in by_len.items():
        run = [gs[0]]
        for g in gs[1:]:
            if len(run) == 1 or g - run[-1] == run[1] - run[0]:
                run.append(g)
            else:
                runs.append((p, run))
                run = [g]
        runs.append((p, run))
    return [(p, r[0], r[1] - r[0] if len(r) > 1 else 1, r) for p, r in runs]


def run_beam_search(step, prefill, reorder, tokens, prompt_lengths, n_query, *, groups, beam_size, num_return_gen,
                    stop_token, tokens_to_generate, max_position_embeddings):
    """DistributedGPT3.beam_search's loop (:1743-1875) for N clips (tokens [N, L], one prompt length per clip) over a
    decode state of `groups` slot groups of beam_size rows each (group g owns rows g*beam .. g*beam + beam - 1), filled
    with clips in input order.  Each clip keeps its own context length, ranking, BeamHypotheses and stopping rule, so
    its result does not depend on the other clips or on `groups`.  When a group's clip is done (its pool is done or its
    own last position is reached) the next waiting clip is prefilled into that group while the other groups keep
    decoding; a group with no successor is frozen.
      prefill(first_group, group_stride, clips, n) -> logits [len(clips), V]: clip clips[i]'s [prefix | tokens[:n]] into
        group first_group + i * group_stride (refills of one step with one prompt length and equally spaced groups
        share a call);
      step(new_tokens [groups*beam, 1], live [groups] bools) -> logits [groups*beam, V] of one single-token step (the
        rows of a group that is not live are never read);
      reorder(idx [groups*beam]) permutes the decode state's rows (within groups).
    A decoding step ranks every live group's candidates in one device sort, copies them to the host in one transfer and
    applies the survivors with one host-to-device copy; the step that starts clips ranks their first candidates (one
    beam per clip: its beams are identical) in one more of each.  Returns a list of N AttrDict(sequences, scores) in
    input order."""
    N, dev = tokens.size(0), tokens.device
    plens = [int(p) for p in prompt_lengths]
    assert len(plens) == N
    tokens = torch.cat((tokens, torch.full((N, tokens_to_generate), stop_token, dtype=torch.long, device=dev)), dim=-1)
    final_len = min(tokens.size(1), max_position_embeddings)
    if max(plens) >= final_len:
        raise ValueError('context length + tokens_to_generate too large')
    G, beam, top, width = groups, beam_size, 2 * beam_size, tokens.size(1)
    clip_of = [None] * G        # clip decoding in group g (None: free / frozen)
    ctx = [0] * G               # the group's next context position
    pools = [None] * G
    out = [None] * N
    rows = torch.full((G * beam, width), stop_token, dtype=torch.long, device=dev)
    scores = torch.zeros(G * beam, 1, dtype=torch.float32, device=dev)
    new = torch.full((G * beam, 1), stop_token, dtype=torch.long, device=dev)   # each row's next input token
    waiting = list(range(N))

    def finish(g, add):
        c, pool, base = clip_of[g], pools[g], g * beam
        if add:   # the clip reached its last position without being done: its live beams join the pool
            for b in range(beam):
                pool.add(rows[base + b].clone(), scores[base + b], ctx[g] + 1 - plens[c])
        best = sorted(pool.beams, key=lambda x: float(x[0]), reverse=True)[:min(num_return_gen, len(pool.beams))]
        out[c] = AttrDict(sequences=torch.stack([h for _, h, _ in best], dim=0),
                          scores=torch.stack([torch.as_tensor(sc, device=dev).reshape(-1)[0] for sc, _, _ in best], dim=0))
        clip_of[g] = None

    def rank(gs, cand, vocab, gather):
        """Rank the clips of groups gs from cand [len(gs), width] (one sort, one transfer), write the survivors of the
        groups that go on into rows / scores / new (one transfer), advance or finish each group.  gather: the survivors
        may come from any beam of their group (a decoding step; otherwise they all come from the group's identical
        beams): every row is gathered from its source row first, and that index (identity for the other groups) is
        returned for the reorder."""
        nonlocal rows
        ranked_scores, ranked = torch.sort(cand, dim=-1, descending=True)
        ranked, ranked_scores = ranked[:, :top], ranked_scores[:, :top]
        host = torch.cat((ranked.double(), ranked_scores.double()), dim=1).cpu()   # indices < 2**53 and fp32 are exact
        idx = host[:, :top].long()
        beam_of, word_of = torch.div(idx, vocab, rounding_mode='floor').tolist(), (idx % vocab).tolist()
        best_score = host[:, top:].max(dim=1).values.tolist()
        keep, going, words, picked = list(range(G * beam)), [], [], []
        for i, g in enumerate(gs):
            c, base = clip_of[g], g * beam
            survivors = []
            for r, (word, b) in enumerate(zip(word_of[i], beam_of[i])):
                if word == stop_token:
                    if r >= beam:  # a finished hypothesis outside the top beam_size candidates is dropped
                        continue
                    pools[g].add(rows[base + b].clone(), ranked_scores[i, r], ctx[g] + 1 - plens[c])
                else:
                    survivors.append((word, r, b))
                if len(survivors) == beam:
                    break
            if pools[g].is_done(best_score[i], ctx[g] + 1 - plens[c]):
                finish(g, False)
                continue
            going.append(g)
            keep[base:base + beam] = [base + b for _, _, b in survivors]
            words += [w for w, _, _ in survivors]
            picked += [i * top + r for _, r, _ in survivors]
        if not going:
            return None
        dst = [g * beam + j for g in going for j in range(beam)]
        at = [r * width + ctx[r // beam] for r in dst]
        head = keep if gather else []
        keep, dst, words, picked, at = torch.tensor(head + dst + words + picked + at, dtype=torch.long,
                                                    device=dev).split([len(head)] + [len(dst)] * 4)
        if gather:
            rows = rows.index_select(0, keep)
        rows.view(-1).index_copy_(0, at, words)   # not put_: it fails under torch.use_deterministic_algorithms
        scores.index_copy_(0, dst, ranked_scores.take(picked).view(-1, 1))
        new.index_copy_(0, dst, words.view(-1, 1))
        for g in going:
            if ctx[g] + 1 == final_len:
                finish(g, True)
            ctx[g] += 1
        return keep if gather else None

    def refill(free):
        """Start waiting clips in the free groups (ascending) and rank their first candidates; repeat for clips that
        end at once."""
        while free and waiting:
            gs, cs = free[:len(waiting)], waiting[:len(free)]
            del waiting[:len(gs)]
            for g, c in zip(gs, cs):
                clip_of[g], ctx[g], pools[g] = c, plens[c], BeamHypotheses(beam)
                rows[g * beam:(g + 1) * beam] = tokens[c]
            first = [None] * len(gs)
            for p, g0, gstride, run in _prefill_runs(gs, [plens[c] for c in cs]):
                lg = prefill(g0, gstride, [clip_of[g] for g in run], p)
                for j, g in enumerate(run):
                    first[gs.index(g)] = lg[j:j + 1]
            lg = torch.cat(first)
            rank(gs, torch.log_softmax(lg.float(), dim=-1), lg.size(1), False)
            free = [g for g in gs if clip_of[g] is None]

    refill(list(range(G)))
    while any(c is not None for c in clip_of):
        live = [c is not None for c in clip_of]
        logits = step(new, live)
        gs = [g for g in range(G) if live[g]]
        cand = (torch.log_softmax(logits.float(), dim=-1) + scores).view(G, -1)
        keep = rank(gs, cand if len(gs) == G else cand[gs], logits.size(-1), True)
        if keep is not None:
            reorder(keep)
        refill([g for g in gs if clip_of[g] is None])
    return out


def streams_beam_search(prompt_lengths, beam_size, head_dim, device):
    """Does DistributedGPT3.beam_search run these clips as one streaming search (run_beam_search over the per-row decode
    state, a finished clip's group refilled)?  Only where it gains and its per-sequence decoding step exists: the clips
    need more than one chunk of the batched search (more than 64 // beam_size clips, or several prompt lengths; one
    chunk has nothing to refill), the decoder's head_dim has the per-sequence decode attention (64 / 80 / 96) and the
    tokens are on a CUDA device, where those kernels run.  Otherwise one search per chunk over the fixed-length decode
    state."""
    from ymp import ops
    if torch.device(device).type != "cuda" or head_dim not in (64, 80, 96):
        return False
    return len(beam_search_chunks(prompt_lengths, beam_size, ops.SKINNY_WIDE_MAX_ROWS)) > 1


def beam_search_chunks(prompt_lengths, beam_size, max_rows):
    """How a batched beam search splits its clips: clips grouped by prompt length (in order of first appearance),
    each group cut into chunks of at most max_rows // beam_size clips.  Returns [(prompt_length, [clip indices])]."""
    per = max_rows // beam_size
    if per < 1:
        raise ValueError(f"beam_size {beam_size} exceeds the {max_rows} rows of one decoding step")
    groups = {}
    for i, p in enumerate(prompt_lengths):
        groups.setdefault(int(p), []).append(i)
    return [(p, idx[s:s + per]) for p, idx in groups.items() for s in range(0, len(idx), per)]


class GPT3Model(nn.Module):
    """Parameter container with the reference's names: language_model.{embedding,encoder}...."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        H, F4, V, Lyr = config.hidden_size, config.ffn_hidden_size, config.vocab_size, config.num_hidden_layers
        std = config.init_method_std
        std_out = std / math.sqrt(2.0 * Lyr)

        def n(*shape, s=std):
            return torch.empty(*shape).normal_(0.0, s)

        lm = Holder()
        self.add_module("language_model", lm)
        lm.add_module("embedding", Holder())
        lm.embedding.add_module("word_embeddings", EmbedHolder())
        add_param(lm, "embedding.word_embeddings.weight", n(V, H))
        add_param(lm, "embedding.position_embeddings.weight", n(config.max_position_embeddings, H))
        for i in range(Lyr):
            b = f"encoder.layers.{i}."
            for nm in ("input_layernorm", "post_attention_layernorm"):
                add_param(lm, b + nm + ".weight", torch.ones(H))
                add_param(lm, b + nm + ".bias", torch.zeros(H))
            add_param(lm, b + "self_attention.query_key_value.weight", n(3 * H, H))
            add_param(lm, b + "self_attention.query_key_value.bias", torch.zeros(3 * H))
            add_param(lm, b + "self_attention.dense.weight", n(H, H, s=std_out))
            add_param(lm, b + "self_attention.dense.bias", torch.zeros(H))
            add_param(lm, b + "mlp.dense_h_to_4h.weight", n(F4, H))
            add_param(lm, b + "mlp.dense_h_to_4h.bias", torch.zeros(F4))
            add_param(lm, b + "mlp.dense_4h_to_h.weight", n(H, F4, s=std_out))
            add_param(lm, b + "mlp.dense_4h_to_h.bias", torch.zeros(H))
        add_param(lm, "encoder.final_layernorm.weight", torch.ones(H))
        add_param(lm, "encoder.final_layernorm.bias", torch.zeros(H))

    def word_embeddings_weight(self):
        return self.language_model.embedding.word_embeddings.weight


class DistributedGPT3(nn.Module):
    def __init__(self, model_dir, rank=0, path_load_tag='model', *args, **kwargs):
        super().__init__()
        megatron_cfg = kwargs.pop('megatron_cfg', None)
        _check_tp1(megatron_cfg)
        self.config = GPT3Config.from_pretrained(model_dir)
        # Megatron-LM's name for per-layer activation checkpointing (off by default)
        self.config.checkpoint_activations = bool((megatron_cfg or {}).get('checkpoint_activations', False))
        self.dist_model = GPT3Model(self.config)
        kwargs.pop('checkpoint_model_parallel_size', None)
        if kwargs.pop('load_state_dict', True):
            path = _ckpt_name(0, model_dir, path_load_tag)
            if osp.exists(path):
                self.dist_model.load_state_dict(pre_load(0, model_dir, tag=path_load_tag))
            elif os.environ.get("YMP_ALLOW_RANDOM_INIT", "0") != "1":
                raise FileNotFoundError(f"{path} not found (set YMP_ALLOW_RANDOM_INIT=1 to run with "
                                        "random-initialised decoder weights, e.g. for benchmarks)")
        self.inference_params = None
        self._keys_prefix = "text_decoder.dist_model."

    def train(self, mode=True):
        if mode:
            self.inference_params = None
        return super().train(mode)

    def _param_list(self):
        return named_param_list(self.dist_model, self._keys_prefix)

    def forward(self, tokens=None, input_embeds=None, query_embeds=None, attention_mask=None,
                position_ids=None, labels=None, prompt_length=None, loss_mask=None, is_pair=(False,)):
        """Same contract as the reference (:1578-1618): returns Dict(logits, loss, losses,
        last_hidden_state).  A plain causal mask over the whole sequence and position ids
        arange(S) are always used (the reference never forwards `attention_mask` into the layers
        on this path, :1329-1332), so explicit attention_mask/position_ids are accepted only in
        that default form."""
        if tokens is not None and input_embeds is not None:
            raise ValueError("You cannot specify both decoder_input_ids and decoder_inputs_embeds at the same time")
        if tokens is None and input_embeds is None:
            raise ValueError("You have to specify either decoder_input_ids or decoder_inputs_embeds")
        if position_ids is not None:
            raise NotImplementedError("custom position_ids are not supported on the H100 path")
        if tokens is not None:
            input_embeds = self.dist_model.language_model.embedding.word_embeddings(tokens)
        if query_embeds is not None:
            input_embeds = torch.cat([query_embeds.to(input_embeds.dtype), input_embeds], dim=1)
        if labels is None:
            return self._decode(tokens, input_embeds, 0 if query_embeds is None else query_embeds.size(1))
        keys, params = self._param_list()
        logits, losses, hidden = YF.GptFn.apply(input_embeds, labels.contiguous(), self.config.engine_cfg(self.training), True,
                                                keys, *params)
        if loss_mask is None:
            loss_mask = attention_mask[:, 1:].contiguous()
        losses = losses[:, :-1].contiguous().float()
        lm = loss_mask.reshape(-1).float()
        loss = torch.sum(losses.reshape(-1) * lm) / lm.sum()
        return AttrDict(logits=logits, loss=loss, losses=losses, last_hidden_state=hidden)

    def dropout_active(self):
        """Does a pass in the current mode draw dropout masks (train() mode and a non-zero probability)?"""
        return YF.gpt_dropout_active(self.config.engine_cfg(self.training))

    def text_features(self, tokens, attention_mask):
        """Pooled final hidden states [B, H] of the texts tokens [B, L]: for each text, the final-LayerNorm state of
        column attention_mask.sum(-1) - 1, bit-identical to that row of forward(tokens=...).last_hidden_state.  The texts
        are packed back to back without padding rows (ymp.functional.gpt_text_features) and no LM head is run.  Forward
        only and without dropout."""
        if self.dropout_active():
            raise ValueError("text_features: the decoder's dropout is active (train() mode with p > 0)")
        keys, params = self._param_list()
        return YF.gpt_text_features(tokens, attention_mask, self.config.engine_cfg(self.training), keys, params)

    def prefix_kv(self, query_embeds, lazy=False):
        """Keys and values of the V prefixes query_embeds [V,Q,H] at every decoder layer (ymp.engine.PrefixKV, [layers,
        V*Q, 2H] bf16): pass it to forward_shared_prefix(prefix_kv=...) with the same query_embeds to score any number
        of text batches against these prefixes without computing them again.  Forward only and without dropout.
        lazy: only allocate it; the first forward_shared_prefix that receives it computes the prefixes and fills it."""
        if self.dropout_active():
            raise ValueError("prefix_kv: the decoder's dropout is active (train() mode with p > 0)")
        if lazy:
            from ymp import engine
            V, Q, _ = query_embeds.shape
            return engine.PrefixKV.empty(self.config.engine_cfg(self.training), V, Q, query_embeds.device)
        keys, params = self._param_list()
        return YF.gpt_prefix_kv(query_embeds, self.config.engine_cfg(self.training), keys, params)

    def forward_shared_prefix(self, query_embeds, input_embeds, labels=None, hidden_rows=None, shared_cols=None,
                              used_cols=None, prefix_kv=None):
        """Score N = V*t texts against V visual prefixes without repeating them: text n follows prefix n // t under the
        same plain causal mask as forward() on torch.cat([query_embeds.repeat_interleave(t, 0), input_embeds], 1).
        query_embeds [V,Q,H], input_embeds [N,L,H]; labels [N,L] are the targets of the text positions.
        shared_cols: per-video count of leading text columns all t texts of the video have in common (a title prompt),
        computed once per video; used_cols: per-video count of text columns its texts use (default L).  See
        ymp.functional.gpt_shared_prefix for which columns are then computed; the others read +0.
        Forward only and without dropout (evaluation): returns Dict(losses [N,L] fp32 per-token CE of the text
        positions or None, hidden [len(hidden_rows), H] final hidden states of text rows n*L + j or None), each value
        bit-identical to the matching position of forward() on the repeated layout.
        prefix_kv: the handle prefix_kv(query_embeds) returned for these query_embeds; the prefixes are then not
        computed at all.  A handle whose V, Q, H or layer count differs from the call's is rejected."""
        if self.dropout_active():
            raise ValueError("forward_shared_prefix: the decoder's dropout is active (train() mode with p > 0)")
        keys, params = self._param_list()
        losses, hidden = YF.gpt_shared_prefix(query_embeds, input_embeds.to(query_embeds.dtype), labels, hidden_rows,
                                              self.config.engine_cfg(self.training), keys, params, shared=shared_cols,
                                              used=used_cols, prefix_kv=prefix_kv)
        return AttrDict(losses=losses, hidden=hidden)

    # ------------------------------------------------------------------------------------------ generation
    def _decode(self, tokens, input_embeds, n_query):
        """Inference branch of forward (:1576-1603): one incremental step over the KV cache.  input_embeds
        [B, n, H] already holds [prefix | word embeddings]; logits are returned for the LAST position only
        ([B, 1, V] fp32 - the only row sample()/beam_search() read)."""
        from ymp import engine, ops
        if self.inference_params is None:
            raise ValueError("no labels and no inference_params: call sample()/beam_search()/generate()")
        ip = self.inference_params
        B, n, H = input_embeds.shape
        ts = ip.token_step
        if ts is not None and n == 1:
            # steady state of sample() / beam_search(): nothing but the graph replay on the host path (walking the module
            # tree for the parameter list alone costs more than the whole device step; weights cannot change inside
            # one generate call - the step object was validated when this call acquired its cache)
            hid, logits = ts.run(input_embeds.reshape(B, H))
            ip.sequence_len_offset += 1
            return AttrDict(logits=logits.view(B, 1, -1), loss=None, losses=None, last_hidden_state=hid.view(B, 1, H))
        keys, params = self._param_list()
        if ip.cache is None:
            ip.cache = self._resident_cache(ip.max_batch_size, ip.max_sequence_len, input_embeds.device, per_row=False)
            ip.cache.reset()
            ip.key_value_memory_dict = {i + 1: t for i, t in enumerate(ip.cache.qkv)}
        off = ip.sequence_len_offset
        stride = ip.prefill_stride if off == 0 else 1
        assert off == ip.cache.len and B * stride == ip.cache.B
        if n == 1 and off > 0 and B <= (ops.SKINNY_WIDE_MAX_ROWS if ip.wide_step else ops.SKINNY_MAX_ROWS):
            # single-token step: skinny GEMMs + device-side cache length, replayed as one CUDA graph
            ts = self._token_step(ip.cache, keys, params, input_embeds.dtype, per_row=False)
            if ts.static:
                ip.token_step = ts
            hid, logits = ts.run(input_embeds.reshape(B, H))
        else:
            W = {k: YF.as_bf16(p) for k, p in zip(keys, params)}
            pos = W[engine.GPT + "embedding.position_embeddings.weight"]
            x = (input_embeds.float() + pos[off:off + n][None].float()).reshape(B * n, H).contiguous()
            hid = engine.gpt_decode(W, x, ip.cache, n, seq_stride=stride)
            logits = ops.gemm(hid, W[engine.GPT + "embedding.word_embeddings.weight"]).float()
        ip.sequence_len_offset += n  # tokens.size(1) + query_embeds.size(1) of the reference
        return AttrDict(logits=logits.view(B, 1, -1), loss=None, losses=None, last_hidden_state=hid.view(B, 1, H))

    def _resident_cache(self, batch, max_len, device, per_row):
        """The KV cache of `batch` sequences x max_len positions for one length mode (per_row: ymp.engine.KVCache's
        per-sequence lengths, else its one scalar length).  It is kept on the model with its captured token step and
        reused by later sample() / beam_search() calls: caption evaluation decodes thousands of clips with the same
        shape.  One shape stays resident (a 1.3B cache at beam 5 x 400 positions is 0.6 GB)."""
        from ymp import engine
        key = (batch, max_len, str(device), per_row)
        pool = self.__dict__.setdefault("_decode_pool", {})
        if key not in pool:
            pool.clear()
            pool[key] = engine.KVCache(self.config.engine_cfg(), batch, max_len, device)
        return pool[key]

    def _token_step(self, cache, keys, params, emb_dtype, per_row):
        """cache's single-token step (ymp.engine.TokenStep) for the weights `params`: rebuilt when they moved or changed
        version.  The graph may hold raw pointers to bf16 parameters (used in place) and frozen fp32 ones (their bf16
        copy is cached until the version changes); trainable fp32 ones are re-cast on every call."""
        from ymp import engine
        sig = (params[0].data_ptr(), params[-1].data_ptr(), sum(p._version for p in params))
        ts = cache.token
        if ts is None or ts.sig != sig or ts.per_row != per_row:
            static = all(p.dtype == torch.bfloat16 or not p.requires_grad for p in params)
            ts = cache.token = engine.TokenStep(cache, {k: YF.as_bf16(p) for k, p in zip(keys, params)}, emb_dtype, sig,
                                                static, per_row=per_row)
        elif not ts.static:
            ts.W = {k: YF.as_bf16(p) for k, p in zip(keys, params)}
        return ts

    def _decode_callbacks(self, query_embeds):
        def step(new_tokens, first):
            out = self(tokens=new_tokens, query_embeds=query_embeds if first else None)
            return out.logits[:, -1, :]

        def reorder(idx):
            # the beam loops own the cache: permute the row table the decoding steps read keys through, move no K/V
            # row (swap_key_value_dict keeps the reference's physical permutation)
            self.inference_params.cache.reindex(idx)
        return step, reorder

    def _fixed_len_decoder(self, tokens, query_embeds, groups, beam_size, max_len, wide):
        """run_beam_search's decode state over a KV cache with one length for all rows (InferenceParams + _decode,
        through _decode_callbacks): the clips tokens [groups, L] start together at one prompt length and step together;
        a finished clip's rows keep stepping unread.  wide: the chunked search's form (the prefill runs each clip's
        [prefix | prompt] once, into its first beam slot, and the cache's row table points the clip's other beams at it;
        single-token steps of up to 64 rows take the captured step); otherwise one clip whose prefill runs beam_size
        identical rows.  Returns (step, prefill, reorder)."""
        assert wide or groups == 1
        ip = self.inference_params = InferenceParams(groups * beam_size, max_len)
        ip.wide_step, ip.prefill_stride = wide, beam_size if wide else 1
        qe = query_embeds if wide or query_embeds is None else query_embeds.repeat(beam_size, 1, 1)
        step, reorder = self._decode_callbacks(qe)

        def prefill(group0, group_stride, clips, n):
            assert ip.sequence_len_offset == 0, "the fixed-length decode state is prefilled once"
            assert group0 == 0 and group_stride == 1 and list(clips) == list(range(groups))
            if wide:
                return step(tokens[:, :n], True)
            return step(tokens[:, :n].repeat(beam_size, 1), True)[:1]
        return (lambda new_tokens, live: step(new_tokens, False)), prefill, reorder

    def _per_row_decoder(self, tokens, query_embeds, groups, beam_size, max_len):
        """run_beam_search's decode state over a KV cache in per-row mode: each group at its own length, the
        single-token steps replay one captured per-row TokenStep that advances the live groups' rows only, and a
        finished clip's group is refilled by a group prefill into its first slot.  Returns (step, prefill, reorder)."""
        from ymp import engine, ops
        rows, dev = groups * beam_size, tokens.device
        nq = 0 if query_embeds is None else query_embeds.size(1)
        self.inference_params = None
        cache = self._resident_cache(rows, max_len, dev, per_row=True)
        cache.reset_rows()
        emb = self.dist_model.language_model.embedding.word_embeddings
        ts = self._token_step(cache, *self._param_list(), emb.weight.dtype, per_row=True)
        W = ts.W
        wemb, pos = W[engine.GPT + "embedding.word_embeddings.weight"], W[engine.GPT + "embedding.position_embeddings.weight"]

        def step(new_tokens, live):
            cache.set_live([x for x in live for _ in range(beam_size)])
            _, logits = ts.run(emb(new_tokens).reshape(rows, -1))
            return logits

        def prefill(group0, group_stride, clips, n):
            sel = torch.tensor(clips, dtype=torch.long, device=dev)
            x = emb(tokens[sel, :n])
            if query_embeds is not None:
                x = torch.cat([query_embeds[sel].to(x.dtype), x], dim=1)
            m = n + nq
            x = (x.float() + pos[:m][None].float()).reshape(len(clips) * m, -1).contiguous()
            hid = cache.prefill_groups(W, x, m, group0, group_stride, beam_size)
            return ops.gemm(hid, wemb).float()
        return step, prefill, cache.reindex_rows

    @torch.no_grad()
    def sample(self, tokens, query_embeds=None, temperature=1.0, use_eod_token_for_early_termination=True,
               stop_on_double_eol=False, stop_on_eol=False, termination_id=None, **kwargs):
        """Batched greedy / top-k / top-p decoding (:1620-1741)."""
        cfg = self.config
        lengths = kwargs.pop('prompt_length', torch.tensor([tokens.size(1)], device=tokens.device))
        lengths = torch.as_tensor(lengths, device=tokens.device).reshape(-1)
        nq = 0 if query_embeds is None else query_embeds.size(1)
        max_len = min(tokens.size(1) + cfg.tokens_to_generate, cfg.max_position_embeddings)
        self.inference_params = InferenceParams(tokens.size(0), max_len + nq)
        step, _ = self._decode_callbacks(query_embeds)
        return run_sample(step, tokens, lengths, nq, tokens_to_generate=cfg.tokens_to_generate, eod_id=cfg.eod_id,
                          max_position_embeddings=cfg.max_position_embeddings, top_k=cfg.top_k, top_p=cfg.top_p,
                          temperature=temperature, vocab_size=cfg.vocab_size, termination_id=termination_id,
                          use_eod_token_for_early_termination=use_eod_token_for_early_termination,
                          stop_on_double_eol=stop_on_double_eol, stop_on_eol=stop_on_eol)

    @torch.no_grad()
    def beam_search(self, tokens, query_embeds=None, beam_size=5, num_return_gen=1, stop_token=None, **kwargs):
        """Beam search (:1743-1875) through run_beam_search.  One sample (tokens [1, L]): Dict(sequences [n, len],
        scores [n]), over the fixed-length decode state.  B > 1 samples (prompt_length an int or a [B] tensor): a list
        of B such Dicts, each equal to the call for that sample alone.  Samples that need more than one chunk run one
        streaming search over the per-row decode state (_beam_search_stream: a finished sample's beam slots take the
        next sample) where streams_beam_search says so; otherwise one search per chunk of samples that share a prompt
        length (_beam_search_batched)."""
        cfg = self.config
        prompt_length = kwargs.pop('prompt_length', tokens.size(1))
        if stop_token is None:
            stop_token = cfg.eod_id
        if tokens.size(0) > 1:
            lengths, _, _, _ = self._beam_search_args(tokens, query_embeds, prompt_length, beam_size, num_return_gen, stop_token)
            stream = streams_beam_search(lengths, beam_size, cfg.hidden_size // cfg.num_attention_heads, tokens.device)
            search = self._beam_search_stream if stream else self._beam_search_batched
            return search(tokens, query_embeds, beam_size, num_return_gen, stop_token, prompt_length)
        lengths, nq, max_len, kw = self._beam_search_args(tokens, query_embeds, prompt_length, beam_size, num_return_gen,
                                                          stop_token)
        dec = self._fixed_len_decoder(tokens, query_embeds, 1, beam_size, max_len, wide=False)
        return run_beam_search(*dec, tokens, lengths, nq, groups=1, **kw)[0]

    def _beam_search_args(self, tokens, query_embeds, prompt_length, beam_size, num_return_gen, stop_token):
        """(one prompt length per sample, prefix length, KV-cache length, run_beam_search's keyword arguments)."""
        cfg = self.config
        lengths = torch.as_tensor(prompt_length).reshape(-1).tolist()
        lengths = lengths * tokens.size(0) if len(lengths) == 1 else lengths
        assert len(lengths) == tokens.size(0)
        nq = 0 if query_embeds is None else query_embeds.size(1)
        max_len = min(tokens.size(1) + cfg.tokens_to_generate, cfg.max_position_embeddings) + nq
        return lengths, nq, max_len, dict(beam_size=beam_size, num_return_gen=num_return_gen, stop_token=stop_token,
                                          tokens_to_generate=cfg.tokens_to_generate,
                                          max_position_embeddings=cfg.max_position_embeddings)

    def _beam_search_batched(self, tokens, query_embeds, beam_size, num_return_gen, stop_token, prompt_length):
        """run_beam_search per chunk of beam_search_chunks (clips of one prompt length), one group per clip of a
        fixed-length decode state."""
        from ymp import ops
        lengths, nq, max_len, kw = self._beam_search_args(tokens, query_embeds, prompt_length, beam_size, num_return_gen,
                                                          stop_token)
        res = [None] * tokens.size(0)
        for plen, clips in beam_search_chunks(lengths, beam_size, ops.SKINNY_WIDE_MAX_ROWS):
            sel = torch.tensor(clips, dtype=torch.long, device=tokens.device)
            toks, qe = tokens[sel], None if query_embeds is None else query_embeds[sel]
            dec = self._fixed_len_decoder(toks, qe, len(clips), beam_size, max_len, wide=True)
            for i, o in zip(clips, run_beam_search(*dec, toks, [plen] * len(clips), nq, groups=len(clips), **kw)):
                res[i] = o
        return res

    def _beam_search_stream(self, tokens, query_embeds, beam_size, num_return_gen, stop_token, prompt_length):
        """One run_beam_search over all clips in G = 64 // beam_size groups of a per-row decode state."""
        from ymp import ops
        lengths, nq, max_len, kw = self._beam_search_args(tokens, query_embeds, prompt_length, beam_size, num_return_gen,
                                                          stop_token)
        G = min(ops.SKINNY_WIDE_MAX_ROWS // beam_size, tokens.size(0))
        dec = self._per_row_decoder(tokens, query_embeds, G, beam_size, max_len)
        return run_beam_search(*dec, tokens, lengths, nq, groups=G, **kw)

    @torch.no_grad()
    def generate(self, tokens, do_sample=True, termination_id=None, *args, **kwargs):
        """(:1878-1883)"""
        if do_sample:
            return self.sample(tokens, termination_id=termination_id, *args, **kwargs)
        return self.beam_search(tokens, stop_token=termination_id, *args, **kwargs)
