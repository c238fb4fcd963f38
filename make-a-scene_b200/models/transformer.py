"""Drop-in for reference models/transformer.py (MakeAScene token transformer, tier 2) on the sm_90a kernels.

Same class names, constructor signatures, attribute names and state_dict keys (including the `transformer.mask`
buffer). Supported configuration = the reference's defaults: cogview_pb_relax=True (a softmax-invariant shift),
sandwich LayerNorm, no prescale, no rudalle_relax; attention and residual dropout at any 0 <= p <= 1 (masks generated inside
the kernels, include/mas_b200.h). The reference's `cache` / `use_cache` arguments raise
(its cache path is broken: transformer.py:73 vs :181, SURVEY.md 3.5); autoregressive sampling with a KV cache and
classifier-free guidance is `MakeAScene.generate` (new API, SURVEY.md 8f-3: specified by the non-cached forward).
Anything else raises — there is no fallback path.
"""
import math

import torch
import torch.nn as nn

from mas_b200 import ops


def gelu(x):
    """OpenAI tanh-GELU, transformer.py:11-14."""
    return ops.GeluFn.apply(x)


class LayerNorm(nn.LayerNorm):
    def forward(self, x, residual=None, p=0.0):
        """LN(x) + residual; p > 0: LN(dropout_p(x)) + residual in one kernel (the sandwich LayerNorm after a dropout site)."""
        return ops.LayerNormFn.apply(x, self.weight, self.bias, residual, self.eps, p)


class Linear(nn.Linear):
    """fp8: a plain attribute (not a parameter or buffer, so the state_dict is unchanged). True runs the layer's training calls on
    the FP8 kernels (ops.linear: only calls that record an autograd graph, only where ops.linear_fp8_on holds); every other call
    runs exactly as with False. MakeAScene(fp8_linear=True) sets it on the four Linear layers of every TransformerLayer."""
    fp8 = False

    def forward(self, x):
        return ops.linear(x, self.weight, self.bias, self.fp8)


def _drop_p(mod):
    """The probability a dropout holder (nn.Dropout) applies now: its .p in training mode, 0 in eval mode."""
    if not mod.training:
        return 0.0
    p = float(mod.p)
    if not 0.0 <= p <= 1.0:
        raise ValueError("dropout probability has to be between 0 and 1, but got %r" % (mod.p,))
    return p


def _dropout(x, mod, residual=None):
    """residual + dropout(x) with the holder's current probability (the torch add when nothing is dropped)."""
    p = _drop_p(mod)
    if p > 0:
        return ops.DropoutFn.apply(x, p, residual)
    return x if residual is None else residual + x


class SelfAttention(nn.Module):
    def __init__(self, hidden_dim, num_attn_heads, attn_dropout_prob, out_dropout_prob, cogview_pb_relax=True, rudalle_relax=False,
                 recompute_attention=False):
        """recompute_attention: the attention stores no S x S probabilities for the backward and recomputes them there
        (ops.CausalAttentionFn(recompute=True)); less memory for more arithmetic. Needs head dim 64 or 128 and S % 128 == 0."""
        super().__init__()
        self.recompute_attention = recompute_attention
        self.hidden_dim = hidden_dim
        self.num_attn_heads = num_attn_heads
        self.d = math.sqrt(self.hidden_dim // self.num_attn_heads)
        self.qkv = Linear(hidden_dim, 3 * hidden_dim)
        self.attn_drop = nn.Dropout(attn_dropout_prob)
        self.out_proj = Linear(hidden_dim, hidden_dim)
        self.out_drop = nn.Dropout(out_dropout_prob)
        self.cogview_pb_relax = cogview_pb_relax
        self.rudalle_relax = rudalle_relax
        if rudalle_relax:
            raise NotImplementedError("rudalle_relax has no kernel (reference default is off)")

    def forward(self, x, mask=None, use_cache=False, cache=None):
        if use_cache or cache is not None:
            raise NotImplementedError("KV cache: the reference path is broken (transformer.py:73 vs :181); no kernel")
        return _dropout(self.project(x), self.out_drop), None

    def project(self, x):
        """out_proj(attention) with attention dropout, before out_drop (TransformerLayer fuses out_drop into the next kernel)."""
        return self.out_proj(ops.CausalAttentionFn.apply(self.qkv(x), self.num_attn_heads, _drop_p(self.attn_drop),
                                                          self.recompute_attention))


class MLP(nn.Module):
    def __init__(self, hidden_dim, dropout_prob, rudalle_relax=False):
        super().__init__()
        self.lin1 = Linear(hidden_dim, 4 * hidden_dim)
        self.lin2 = Linear(4 * hidden_dim, hidden_dim)
        self.dropout = nn.Dropout(dropout_prob)
        self.rudalle_relax = rudalle_relax
        if rudalle_relax:
            raise NotImplementedError("rudalle_relax has no kernel")

    def forward(self, x):
        return _dropout(self.project(x), self.dropout)

    def project(self, x):
        """lin2(gelu(lin1(x))), before the dropout (TransformerLayer fuses it into the next kernel)."""
        return self.lin2(gelu(self.lin1(x)))


class TransformerLayer(nn.Module):
    def __init__(self, hidden_dim, num_attn_heads, attn_dropout_prop, out_dropout_prob, cogview_pb_relax=True,
                 cogview_sandwich_layernorm=True, cogview_layernorm_prescale=False, rudalle_relax=False, recompute_attention=False):
        super().__init__()
        self.cogview_pb_relax = cogview_pb_relax
        self.cogview_sandwich_layernorm = cogview_sandwich_layernorm
        self.cogview_layernorm_prescale = cogview_layernorm_prescale
        self.rudalle_relax = rudalle_relax
        if cogview_layernorm_prescale or rudalle_relax:
            raise NotImplementedError("layernorm prescale / rudalle_relax have no kernel")
        self.ln_in = LayerNorm(hidden_dim, eps=1e-5)
        self.ln_out = LayerNorm(hidden_dim, eps=1e-5)
        if cogview_sandwich_layernorm:
            self.first_ln_sandwich = LayerNorm(hidden_dim, eps=1e-5)
            self.second_ln_sandwich = LayerNorm(hidden_dim, eps=1e-5)
        self.attn = SelfAttention(hidden_dim=hidden_dim, num_attn_heads=num_attn_heads, attn_dropout_prob=attn_dropout_prop,
                                  out_dropout_prob=out_dropout_prob, cogview_pb_relax=cogview_pb_relax, rudalle_relax=rudalle_relax,
                                  recompute_attention=recompute_attention)
        self.mlp = MLP(hidden_dim=hidden_dim, dropout_prob=out_dropout_prob, rudalle_relax=rudalle_relax)

    def forward(self, x, mask=None, cache=None, use_cache=False, mlp_cache=False):
        if use_cache or cache is not None:
            raise NotImplementedError("KV cache has no kernel")
        # out_drop and mlp.dropout act where the reference applies them (transformer.py:114, 139), fused into the kernel that
        # consumes their output: the sandwich LayerNorm (mask applied on load) or, without it, the residual add (mas_dropout)
        attn_out = self.attn.project(self.ln_in(x))
        if self.cogview_sandwich_layernorm:
            x = self.first_ln_sandwich(attn_out, residual=x, p=_drop_p(self.attn.out_drop))      # x + LN(dropout(attn_out)), fused
        else:
            x = _dropout(attn_out, self.attn.out_drop, residual=x)
        mlp_out = self.mlp.project(self.ln_out(x))
        if self.cogview_sandwich_layernorm:
            x = self.second_ln_sandwich(mlp_out, residual=x, p=_drop_p(self.mlp.dropout))
        else:
            x = _dropout(mlp_out, self.mlp.dropout, residual=x)
        return x, None


class Transformer(nn.Module):
    def __init__(self, num_layers, hidden_dim, num_attn_heads, image_tokens_per_dim, seg_tokens_per_dim, text_length,
                 attn_dropout_prop=0, out_dropout_prob=0, cogview_pb_relax=True, cogview_sandwich_layernorm=True,
                 cogview_layernorm_prescale=False, rudalle_relax=False, recompute_attention=False, fp8_linear=False):
        """fp8_linear: see MakeAScene."""
        super().__init__()
        if not isinstance(fp8_linear, bool):
            raise ValueError("fp8_linear must be a bool, got %r" % (fp8_linear,))
        self.num_layers = num_layers
        self.cogview_pb_relax = cogview_pb_relax
        self.rudalle_relax = rudalle_relax
        self.layers = nn.ModuleList([
            TransformerLayer(hidden_dim, num_attn_heads, attn_dropout_prop, out_dropout_prob, cogview_pb_relax,
                             cogview_sandwich_layernorm, cogview_layernorm_prescale, rudalle_relax, recompute_attention)
            for _ in range(num_layers)])
        for layer in self.layers:
            for lin in (layer.attn.qkv, layer.attn.out_proj, layer.mlp.lin1, layer.mlp.lin2):
                lin.fp8 = fp8_linear
        self.register_buffer("mask", self._create_mask(text_length, seg_tokens_per_dim, image_tokens_per_dim))
        self.final_ln = LayerNorm(hidden_dim, eps=1e-5)

    def _create_mask(self, text_length, seg_tokens_per_dim, image_tokens_per_dim):
        size = text_length + seg_tokens_per_dim ** 2 + image_tokens_per_dim ** 2
        return torch.tril(torch.ones(size, size, dtype=torch.float32))

    def forward(self, x, attn_mask=None, cache=None, use_cache=None):
        # attn_mask * self.mask is plain causal for every mask MakeAScene builds (transformer.py:262-263, 366-370):
        # the kernels implement the causal mask directly.
        if use_cache or cache:
            raise NotImplementedError("KV cache has no kernel")
        if attn_mask is not None:
            S = x.shape[1]
            am = attn_mask.to(self.mask.device, self.mask.dtype)
            while am.dim() > 2:        # [B,1,S,S] / [1,1,S,S] -> [S,S] only if it is the same for every row
                if am.shape[0] != 1 and not bool((am == am[:1]).all()):
                    raise RuntimeError("per-sample attention masks have no kernel (only the causal mask is implemented)")
                am = am[0]
            eff = am[:S, :S] * self.mask[:S, :S]
            if not torch.equal(eff != 0, self.mask[:S, :S] != 0):
                raise RuntimeError("attn_mask * causal mask is not the plain causal mask: only causal attention has a kernel "
                                   "(a padding / prefix mask would silently be ignored otherwise)")
        for layer in self.layers:
            x, _ = layer(x)
        return self.final_ln(x), {}


# score(num_samples=n) computes each prompt's prefix once only from this many candidate rows on (B*n, twice that with
# guidance). Below it both forms are bound by the host's launch rate, and the shared form, with two launches per kernel of a
# layer, is the slower (24 layers, 1024 wide, H100 80GB HBM3 at 700 W: 0.68x at 16 rows, 1.06x at 24, 1.8x from 48;
# tools/bench_score.py). The result is the same bits either way.
SCORE_SHARED_MIN_ROWS = 24


def _param_version(model):
    return tuple((p._version, p.data_ptr()) for p in model.parameters())


def _is_per_row(v):
    """A sampling control given per row (a 1-D tensor or a sequence) rather than one value for the call."""
    return isinstance(v, (list, tuple)) or (isinstance(v, torch.Tensor) and v.dim() > 0)


def _row_values(name, v, n, dev, integer=False):
    """The n per-row values of a sampling control as (fp64 host copy, device tensor fp32 or, integer, int32). A scalar is
    repeated; a 1-D tensor must hold n values of a floating (integer: integer) dtype on dev; a sequence is read on the host.
    ValueError otherwise."""
    if isinstance(v, torch.Tensor) and v.dim() > 0:
        ok = not v.dtype.is_floating_point and not v.dtype.is_complex and v.dtype != torch.bool if integer else v.dtype.is_floating_point
        if v.dim() != 1 or v.shape[0] != n or not ok or v.device != dev:
            raise ValueError("%s: one value per output row expected: a 1-D %s tensor of %d values on %s, got %s %s on %s" % (
                name, "integer" if integer else "floating-point", n, dev, v.dtype, tuple(v.shape), v.device))
        host = v.detach().to("cpu", torch.float64)
    elif isinstance(v, (list, tuple)):
        if len(v) != n or not all(isinstance(x, (int, float)) and not isinstance(x, bool) for x in v) or (
                integer and not all(isinstance(x, int) for x in v)):
            raise ValueError("%s: a sequence of %d %s expected, got %r" % (name, n, "ints" if integer else "numbers", v))
        host = torch.tensor([float(x) for x in v], dtype=torch.float64)
    else:
        host = torch.full((n,), float(v), dtype=torch.float64)
    if integer:
        return host, host.clamp(-2 ** 31, 2 ** 31 - 1).to(torch.int32).to(dev)
    return host, host.to(torch.float32).to(dev)


def _attend_append(qkv, kc, vc, suffix, li, pos):
    """Layer li's attention of this token (qkv [R,3H], stored at position pos) over positions 0..pos: one cache per row, or
    with suffix (num_samples > 1) the prefix cache of the row's prompt followed by the row's own suffix cache."""
    if suffix is None:
        return ops.attn_decode_append(qkv, kc[li], vc[li], pos)
    return ops.attn_decode_shared_append(qkv, kc[li], vc[li], suffix[0][li], suffix[1][li], pos)


class _GraphedDecoder:
    """KV caches + one captured CUDA graph per image position for MakeAScene.generate(use_graphs=True).

    A decode step is ~250 launches of a few microseconds each (24 layers x 10 kernels): launched from Python it is
    host-bound (~22 us per launch). The kernels only depend on the position through launch parameters, so each position
    gets its own graph (captured on first use, replayed in position order afterwards; the graphs share one memory pool).
    The caches are fp32 up to 8 rows and fp16 above (the cache read dominates a step at a few hundred rows).
    Above 8 rows the decode Linears read the fp16 weight images of ops.decode_weight_image: they are built here, before any
    capture, and held by the decoder, so the graphs never record a packing launch and never outlive the images they read.
    `version` records every parameter's version and storage: generate() builds a new decoder when it changes.
    samples > 1 (generate(num_samples=n)): the rows are groups of n samples of one prompt. kc / vc are then prefix caches with
    one row per prompt [rows / n, heads, text + seg length, hd], and `suffix` holds every row's own image-position caches
    [rows, heads, image_length, hd]; the element type still follows the row count."""

    def __init__(self, model, rows, dev, samples=1):
        layers = model.transformer.layers
        heads = layers[0].attn.num_attn_heads
        hd = model.hidden_dim // heads
        self.model, self.rows, self.samples = model, rows, samples
        dt = torch.float32 if rows <= ops.DECODE_F32_ROWS else torch.float16
        if samples == 1:
            self.kc = [torch.empty((rows, heads, model.total_length, hd), dtype=dt, device=dev) for _ in layers]
            self.suffix = None
        else:
            prefix = model.text_length + model.seg_length
            self.kc = [torch.empty((rows // samples, heads, prefix, hd), dtype=dt, device=dev) for _ in layers]
            ks = [torch.empty((rows, heads, model.image_length, hd), dtype=dt, device=dev) for _ in layers]
            self.suffix = (ks, [torch.empty_like(k) for k in ks])
        self.vc = [torch.empty_like(k) for k in self.kc]
        self.version = _param_version(model)
        self.images = []
        if rows > ops.DECODE_F32_ROWS:
            lins = [m for l in layers for m in (l.attn.qkv, l.attn.out_proj, l.mlp.lin1, l.mlp.lin2)] + [model.to_logits[1]]
            self.images = [ops.decode_weight_image(m.weight) for m in lins if m.weight.shape[1] % 64 == 0]
        self.tok = torch.zeros(rows, dtype=torch.long, device=dev)
        self.pool = torch.cuda.graph_pool_handle()
        self.graphs, self.keep = {}, {}

    def eager_step(self, t, tok_all, prefix):
        m = self.model
        dev, ip, R = tok_all.device, m.image_tokens_per_dim, self.rows
        row = torch.full((1,), t // ip, dtype=torch.long, device=dev)
        col = torch.full((1,), t % ip, dtype=torch.long, device=dev)
        return self._body(tok_all, row, col, prefix + t)

    def _body(self, tok, row, col, pos):
        m, R = self.model, self.rows
        emb = ops.EmbedFn.apply([(tok.view(R, 1), row, col, 0)], 1, m.hidden_dim, m.image_token_embedding.weight,
                                m.image_row_embeddings.weight, m.image_col_embeddings.weight)
        return m._logits_of(m._decode_step(emb.view(R, m.hidden_dim), self.kc, self.vc, pos, self.suffix), normed=True)

    def graphed_step(self, t, tok_all, prefix):
        self.tok.copy_(tok_all)
        if t not in self.graphs:
            dev, ip = tok_all.device, self.model.image_tokens_per_dim
            row = torch.full((1,), t // ip, dtype=torch.long, device=dev)
            col = torch.full((1,), t % ip, dtype=torch.long, device=dev)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=self.pool):
                out = self._body(self.tok, row, col, prefix + t)
            self.graphs[t], self.keep[t] = g, (out, row, col)
        self.graphs[t].replay()
        return self.keep[t][0]


class MakeAScene(nn.Module):
    def __init__(self, num_layers, hidden_dim, num_attn_heads, image_vocab_size, seg_vocab_size, text_vocab_size,
                 image_tokens_per_dim, seg_tokens_per_dim, text_length, attn_dropout_prob=0.0, out_dropout_prob=0.0,
                 recompute_attention=False, fp8_linear=False):
        """The reference's arguments, plus the dropout probabilities of every layer's attention probabilities
        (attn_dropout_prob) and of its attention and MLP outputs (out_dropout_prob), passed to Transformer; the reference's
        MakeAScene leaves both at 0, which the defaults keep.
        recompute_attention=True: training stores no attention probabilities (S x S per head and sequence) for the backward,
        which recomputes them from per-row statistics; the loss is the same bits, the gradients agree to fp32 rounding.
        Needs head dim 64 or 128 and a sequence length that is a multiple of 128 (RuntimeError otherwise). Not a parameter or
        buffer: the state_dict is unchanged.
        fp8_linear=True: the four Linear layers of every TransformerLayer (attn.qkv, attn.out_proj, mlp.lin1, mlp.lin2) train on
        FP8 tensor cores: e4m3 activations and weights, e5m2 output gradients, one power-of-two scale per tensor from its exact
        max|.| on the device (DESIGN §3.5). It sets the plain attribute `fp8` of those modules (setting `lin.fp8` by hand toggles
        one layer; the state_dict is unchanged). Only calls that record an autograd graph take the FP8 route, so generate, score
        and no-grad forwards return the same bits as with the flag off. to_logits, the embeddings, the LayerNorms and attention
        stay as they are. With the TF32 operand format or MAS_LINEAR_F16=0 the flag has no effect. ValueError unless a bool."""
        super().__init__()
        self.image_tokens_per_dim = image_tokens_per_dim
        self.seg_tokens_per_dim = seg_tokens_per_dim
        self.image_length = image_tokens_per_dim ** 2
        self.seg_length = seg_tokens_per_dim ** 2
        self.text_length = text_length
        self.total_length = self.text_length + self.seg_length + self.image_length
        self.text_vocab_size = text_vocab_size
        self.hidden_dim = hidden_dim
        self.transformer = Transformer(num_layers, hidden_dim, num_attn_heads, image_tokens_per_dim, seg_tokens_per_dim, text_length,
                                       attn_dropout_prob, out_dropout_prob, recompute_attention=recompute_attention,
                                       fp8_linear=fp8_linear)
        self.image_token_embedding = nn.Embedding(image_vocab_size, hidden_dim)
        self.seg_token_embedding = nn.Embedding(seg_vocab_size, hidden_dim)
        self.text_token_embedding = nn.Embedding(text_vocab_size, hidden_dim)
        self.text_pos_embeddings = torch.nn.Embedding(text_length, hidden_dim)
        self.seg_row_embeddings = torch.nn.Embedding(seg_tokens_per_dim, hidden_dim)
        self.seg_col_embeddings = torch.nn.Embedding(seg_tokens_per_dim, hidden_dim)
        self.image_row_embeddings = torch.nn.Embedding(image_tokens_per_dim, hidden_dim)
        self.image_col_embeddings = torch.nn.Embedding(image_tokens_per_dim, hidden_dim)
        for m in (self.text_pos_embeddings, self.seg_row_embeddings, self.seg_col_embeddings, self.image_row_embeddings,
                  self.image_col_embeddings):
            self._init_weights(m)
        self.to_logits = torch.nn.Sequential(LayerNorm(hidden_dim), Linear(hidden_dim, image_vocab_size))

    def reset_sampler(self):
        """Drops the cached KV buffers / CUDA graphs of generate(use_graphs=True) (they are rebuilt by themselves when a
        parameter changes)."""
        self._sampler = None

    def _init_weights(self, module):
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=0.02)
            if isinstance(module, nn.Linear) and module.bias is not None:
                module.bias.data.zero_()
        elif isinstance(module, nn.LayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)

    def _embed(self, text_tokens, seg_tokens, img_tokens):
        """Token + position embeddings of the concatenated sequence, transformer.py:350-364."""
        dev = text_tokens.device
        text_range = torch.arange(self.text_length, device=dev) + (self.text_vocab_size - self.text_length)
        text_tokens = torch.where(text_tokens == 0, text_range, text_tokens)      # pad-id trick, transformer.py:350-353
        ar = lambda n: torch.arange(n, dtype=torch.long, device=dev)
        sp, ip = self.seg_tokens_per_dim, self.image_tokens_per_dim
        segs = [(text_tokens, ar(text_tokens.shape[1]), None, 0),
                (seg_tokens, ar(seg_tokens.shape[1]) // sp, ar(seg_tokens.shape[1]) % sp, text_tokens.shape[1])]
        tables = [self.text_token_embedding.weight, self.text_pos_embeddings.weight, self.text_pos_embeddings.weight,
                  self.seg_token_embedding.weight, self.seg_row_embeddings.weight, self.seg_col_embeddings.weight]
        total = text_tokens.shape[1] + seg_tokens.shape[1]
        if img_tokens is not None:
            segs.append((img_tokens, ar(img_tokens.shape[1]) // ip, ar(img_tokens.shape[1]) % ip, total))
            tables += [self.image_token_embedding.weight, self.image_row_embeddings.weight, self.image_col_embeddings.weight]
            total += img_tokens.shape[1]
        return ops.EmbedFn.apply(segs, total, self.hidden_dim, *tables)

    def forward(self, text_tokens, seg_tokens, img_tokens):
        """Logits [B, image_length, V] predicting every image token from its prefix (transformer.py:366-378). The reference
        computes to_logits over all 640 positions and slices afterwards; LayerNorm and Linear act row by row, so slicing the
        hidden states first gives the same values (and the same, zero, gradient for the dropped rows) at 40 % of the work."""
        emb = self._embed(text_tokens, seg_tokens, img_tokens)
        out, _ = self.transformer(emb)
        out = out[:, -self.image_length - 1:-1, :].contiguous()
        return self.to_logits[1](self.to_logits[0](out))

    def loss(self, text_tokens, seg_tokens, img_tokens):
        """train.py:150-153 in one call: F.cross_entropy(forward(...).view(-1, V), img_tokens.view(-1)) on the fused
        cross-entropy kernels (mas_ce_forward / mas_ce_backward: no log-softmax tensor, the gradient is written once)."""
        return ops.cross_entropy(self.forward(text_tokens, seg_tokens, img_tokens), img_tokens)

    # ---- sampling (SURVEY.md 8f-3) ---------------------------------------------------------------------------
    def _prefill(self, emb, kc=None, vc=None):
        """Full causal pass over emb [B,S,H] with the training kernels and no dropout; returns every position's hidden state
        before final_ln [B,S,H]. With kc / vc (generate's prefix pass) every layer's k / v are recorded at positions 0..S-1.
        Where the fused core runs, the attention writes no probabilities (nothing reads them here): the same outputs."""
        x = emb
        heads = self.transformer.layers[0].attn.num_attn_heads
        stats_only = ops.attn_causal_fused_on(x.shape[1], self.hidden_dim // heads)
        for li, layer in enumerate(self.transformer.layers):
            qkv = layer.attn.qkv(layer.ln_in(x))
            if kc is not None:
                ops.kv_append(qkv, kc[li], vc[li], 0)
            a = layer.attn.out_proj(ops.CausalAttentionFn.apply(qkv, heads, 0.0, stats_only))
            x = layer.first_ln_sandwich(a, residual=x) if layer.cogview_sandwich_layernorm else x + a
            m = layer.mlp.project(layer.ln_out(x))
            x = layer.second_ln_sandwich(m, residual=x) if layer.cogview_sandwich_layernorm else x + m
        return x

    def _score_shares_prefix(self, rows=None):
        """Whether score(num_samples > 1) runs the prefix once per prompt (_prefill_shared): the fused causal core for the
        prefix and the image lengths, the fp16 Linear route for the layers' widths and (when given) at least
        SCORE_SHARED_MIN_ROWS candidate rows. Elsewhere it repeats the prompts."""
        if rows is not None and rows < SCORE_SHARED_MIN_ROWS:
            return False
        heads = self.transformer.layers[0].attn.num_attn_heads
        hd, H = self.hidden_dim // heads, self.hidden_dim
        prefix = self.text_length + self.seg_length
        return (ops.attn_causal_fused_on(prefix, hd) and ops.attn_causal_fused_on(self.image_length, hd)
                and all(ops.linear_f16_on(n, k) for n, k in ((3 * H, H), (H, H), (4 * H, H), (H, 4 * H))))

    def _prefill_shared(self, xp, xs, n):
        """_prefill of prefix rows xp [P,Lp,H] continued by suffix rows xs [P*n,L,H] (row r continues prefix row r // n), in
        lockstep through every layer: each row's hidden states are the bits _prefill gives on the concatenated [P*n,Lp+L,H]
        sequence (prefix rows repeated). Those scale every fp16 operand by max|.| over the whole tensor, prefix rows included,
        so each Linear and attention call here takes the joint maximum of both parts (ops.amax_joint). Returns (xp, xs)."""
        heads = self.transformer.layers[0].attn.num_attn_heads

        def sandwich(ln, a, x):
            return ln(a, residual=x) if ln is not None else x + a
        for layer in self.transformer.layers:
            at, mlp = layer.attn, layer.mlp
            qp, qs = ops.linear_joint([layer.ln_in(xp), layer.ln_in(xs)], at.qkv.weight, at.qkv.bias)
            am = ops.amax_joint(qp, qs)
            cp, cs = ops.attn_causal_given_amax(qp, heads, am), ops.attn_causal_prefix(qp, qs, am, heads)
            ap, as_ = ops.linear_joint([cp, cs], at.out_proj.weight, at.out_proj.bias)
            ln1 = layer.first_ln_sandwich if layer.cogview_sandwich_layernorm else None
            xp, xs = sandwich(ln1, ap, xp), sandwich(ln1, as_, xs)
            mp, ms = ops.linear_joint([layer.ln_out(xp), layer.ln_out(xs)], mlp.lin1.weight, mlp.lin1.bias)
            mp, ms = ops.linear_joint([gelu(mp), gelu(ms)], mlp.lin2.weight, mlp.lin2.bias)
            ln2 = layer.second_ln_sandwich if layer.cogview_sandwich_layernorm else None
            xp, xs = sandwich(ln2, mp, xp), sandwich(ln2, ms, xs)
        return xp, xs

    def _decode_step(self, x, kc, vc, pos, suffix=None):
        """One new token per row (x [R,H], absolute position pos) through all layers against the cache; returns
        final_ln(hidden). Seven launches per layer: qkv, attention (+ cache append), out_proj, the sandwich LayerNorm chained
        with the next input LayerNorm (mas_layernorm2_forward), lin1 (+GELU), lin2, the second chained pair.
        suffix: the per-row caches of _GraphedDecoder when rows share prefix caches (kc / vc) in groups."""
        layers = self.transformer.layers
        if not all(l.cogview_sandwich_layernorm for l in layers) or x.shape[-1] % 4 or x.shape[-1] > 4096:
            return self.transformer.final_ln(self._decode_step_plain(x, kc, vc, pos, suffix))
        y = layers[0].ln_in(x)
        for li, layer in enumerate(layers):
            at, mlp = layer.attn, layer.mlp
            qkv = ops.linear_small(y, at.qkv.weight, at.qkv.bias)
            a = ops.linear_small(_attend_append(qkv, kc, vc, suffix, li, pos), at.out_proj.weight, at.out_proj.bias)
            x, y = ops.layernorm2(a, layer.first_ln_sandwich, x, layer.ln_out)        # x + LN(a), then the MLP's input norm
            m = ops.linear_small(y, mlp.lin1.weight, mlp.lin1.bias, act=1)
            m = ops.linear_small(m, mlp.lin2.weight, mlp.lin2.bias)
            nxt = layers[li + 1].ln_in if li + 1 < len(layers) else self.transformer.final_ln
            x, y = ops.layernorm2(m, layer.second_ln_sandwich, x, nxt)
        return y

    def _decode_step_plain(self, x, kc, vc, pos, suffix=None):
        """The unfused form (configurations without the sandwich LayerNorm); returns the hidden state before final_ln."""
        for li, layer in enumerate(self.transformer.layers):
            at, mlp = layer.attn, layer.mlp
            qkv = ops.linear_small(layer.ln_in(x), at.qkv.weight, at.qkv.bias)
            if suffix is None:
                ops.kv_append(qkv.view(qkv.shape[0], 1, -1), kc[li], vc[li], pos)
                ctx = ops.attn_decode(qkv, kc[li], vc[li], pos + 1)
            else:   # the same two steps on the split caches: the append entry would add this token's term in another order
                ops.kv_append(qkv.view(qkv.shape[0], 1, -1), suffix[0][li], suffix[1][li], pos - kc[li].shape[2])
                ctx = ops.attn_decode_shared(qkv, kc[li], vc[li], suffix[0][li], suffix[1][li], pos + 1)
            a = ops.linear_small(ctx, at.out_proj.weight, at.out_proj.bias)
            x = layer.first_ln_sandwich(a, residual=x) if layer.cogview_sandwich_layernorm else x + a
            m = ops.linear_small(layer.ln_out(x), mlp.lin1.weight, mlp.lin1.bias, act=1)
            m = ops.linear_small(m, mlp.lin2.weight, mlp.lin2.bias)
            x = layer.second_ln_sandwich(m, residual=x) if layer.cogview_sandwich_layernorm else x + m
        return x

    def _logits_of(self, hidden, normed=False):
        """to_logits on hidden states [R,H]; normed: final_ln has been applied already (decode steps)."""
        f = hidden if normed else self.transformer.final_ln(hidden)
        h = self.to_logits[0](f)
        return ops.linear_small(h, self.to_logits[1].weight, self.to_logits[1].bias)

    @torch.no_grad()
    def generate(self, text_tokens, seg_tokens, guidance_scale=None, uncond_text_tokens=None, temperature=1.0, top_k=None,
                 generator=None, img_tokens=None, return_logits=False, use_graphs=False, top_p=None, img_mask=None, num_samples=1,
                 return_logprobs=False, seeds=None):
        """Autoregressive sampling of the image tokens with a KV cache; optional classifier-free guidance
        (logits = uncond + scale * (cond - uncond), the unconditional stream sees padded text; Make-A-Scene paper 3.4).

        text_tokens [B,text_length], seg_tokens [B,seg_length] int64. A call decodes R = B rows (2B with guidance); memory is
        the only limit on R. Up to 8 rows the decode steps are strict fp32 (weights and KV cache). More rows run the decode
        Linear layers on fp16 operands with fp32 accumulation and keep K / V in fp16 caches: the arithmetic of the model's own
        training forward. The prefix pass always runs the training kernels.
        The draw at each position, per row (ru-DALL-E's top_k_top_p_filtering chain, one kernel launch):
          z = logits / temperature; top_k keeps the k largest (ties with the k-th kept); top_p (None or >= 1: off, <= 0:
          ValueError) keeps, of those, every entry whose softmax mass of kept entries with a strictly larger z is <= top_p
          (equal values are kept or dropped together; the largest always stays); the token is the inverse CDF of softmax(z)
          over the kept set at a uniform, in index order. temperature 0 = greedy (the first index of the maximum).
        img_tokens (optional [B,image_length] int64) are fed instead of the sampled ones at every position (teacher forcing —
        what the parity test uses). With img_mask ([B,image_length] bool on the same device) only the positions where it is
        set are forced (image prompts: completion, outpainting, editing a region); the others are drawn, conditioned on all
        earlier tokens, forced or drawn. With guidance a forced token goes to both streams. When sampling with img_mask, the
        B uniforms are drawn at every position, forced or not, so a row's random stream does not depend on the mask: an
        all-false mask gives the tokens of the unprompted call with the same generator.
        Returns tokens [B,image_length] (and the per-position logits [B,image_length,V], mixed and unfiltered, when
        return_logits=True).
        return_logprobs=True also returns logprobs fp32 [B,image_length], last: at a drawn position the natural log of the
        probability the token was drawn with, under the mixed (guided), temperature-scaled, filtered distribution above (the
        draw kernel's own kept-set sum; mas_sample_filtered_logp); 0 at forced positions (img_tokens, or img_mask set) and at
        greedy ones, so a row's sum is the log-probability of its drawn part. Tokens and logits do not depend on the flag.
        The return is then (tokens, logits, logprobs) or (tokens, logprobs).
        num_samples=n (int >= 1) draws n images per prompt: the result is that of generate(text_tokens.repeat_interleave(n, 0),
        seg_tokens.repeat_interleave(n, 0), ...) with the same generator state, bit for bit; output row b*n + j is sample j of
        prompt b, so the returned shapes have B*n rows, and img_tokens / img_mask are given per output row [B*n,image_length]
        (uncond_text_tokens stays per prompt [B,text_length]). The text + segmentation prefix runs once per prompt, its K / V
        are cached once per prompt, and each decode step reads a prompt's prefix once for its group of samples
        (mas_attn_decode_shared_append); the row count R = B*n (2B*n with guidance) still selects fp32 or fp16 decoding.
        use_graphs: replay each position's decode step from a CUDA graph (captured at first use and kept on the module for
        the same row count; captured again after any parameter changes, in place or by replaced storage).
        Dropout is never applied here, in train mode as in eval mode: the prefix pass and the decode steps call the layers'
        kernels directly, not the dropout sites, so a model trained with dropout samples as its eval-mode self.
        Per-row controls: temperature, top_k, top_p and guidance_scale each take one value for the call, or one per output row
        (a 1-D tensor on the model's device, or a sequence, of B*n values; row b*n + j as img_tokens). A row then draws and
        mixes exactly as a call with its values as scalars would (mas_sample_rows / mas_cfg_mix_rows, bit for bit), so one
        call can sweep settings over the samples of a prompt, or batch requests with different settings. ValueError for a
        wrong length, dtype or device, a temperature that is negative or not finite, top_k < 0, top_p <= 0 or a guidance
        scale that is not finite. With per-row scales both streams run for every row unless every scale is 1 (then the call
        is unguided); a row at scale 1 then gets fmaf(1, cond - uncond, uncond), within rounding of its conditional logits
        but not always bitwise equal to them (and the doubled row count may decode in fp16 where the unguided call would not).
        seeds (int64 [B*n] on the model's device; not together with generator): row r draws at image position t with the
        uniform of Philox4x32-10 keyed by seeds[r] at counter t (include/mas_b200.h, mas_sample_rows), which depends on the
        seed and t alone: rows with equal seeds draw with equal uniforms, in this call or another (common random numbers, so
        a sweep compares settings, not noise). Any per-row control or seeds routes the draw to mas_sample_rows; a call with
        scalars only and no seeds issues the entries it always did."""
        B = text_tokens.shape[0]
        dev = text_tokens.device
        n = num_samples
        if isinstance(n, bool) or not isinstance(n, int) or n < 1:
            raise ValueError("num_samples must be an int >= 1, got %r" % (num_samples,))
        if not isinstance(return_logprobs, bool):
            raise ValueError("return_logprobs must be a bool, got %r" % (return_logprobs,))
        Bn = B * n
        if top_p is not None and not _is_per_row(top_p) and not float(top_p) > 0:
            raise ValueError("top_p must be > 0 (None or >= 1: no nucleus filter), got %r" % (top_p,))
        mdev = self.image_token_embedding.weight.device
        rows = None          # per-row draw: (temperature, top_k, top_p) device tensors [B*n]
        if seeds is not None or any(_is_per_row(v) for v in (temperature, top_k, top_p)):
            if seeds is not None:
                if generator is not None:
                    raise ValueError("seeds and generator are two sources of uniforms: pass one of them")
                if not isinstance(seeds, torch.Tensor) or seeds.dtype != torch.int64 or tuple(seeds.shape) != (Bn,) or seeds.device != mdev:
                    raise ValueError("seeds must be an int64 tensor of shape %s on the model's device (%s)" % ((Bn,), mdev))
            temp_h, temp_d = _row_values("temperature", 0.0 if temperature is None else temperature, Bn, mdev)
            topk_h, topk_d = _row_values("top_k", 0 if top_k is None else top_k, Bn, mdev, integer=True)
            topp_h, topp_d = _row_values("top_p", 1.0 if top_p is None else top_p, Bn, mdev)
            if not bool((torch.isfinite(temp_h) & (temp_h >= 0)).all()):
                raise ValueError("temperature must be finite and >= 0 in every row (0: greedy), got %s" % temp_h.tolist())
            if not bool((topk_h >= 0).all()):
                raise ValueError("top_k must be >= 0 in every row (0: off), got %s" % topk_h.tolist())
            if not bool((topp_h > 0).all()):
                raise ValueError("top_p must be > 0 in every row (>= 1: off), got %s" % topp_h.tolist())
            rows = (temp_d, topk_d, topp_d)
            drawing = bool((temp_h > 0).any())
        scale_rows = None    # per-row guidance: fp32 [B*n] device tensor
        if _is_per_row(guidance_scale):
            scale_h, scale_d = _row_values("guidance_scale", guidance_scale, Bn, mdev)
            if not bool(torch.isfinite(scale_h).all()):
                raise ValueError("guidance_scale must be finite in every row, got %s" % scale_h.tolist())
            scale_rows = scale_d if bool((scale_h != 1.0).any()) else None
        if img_tokens is not None and n > 1 and tuple(img_tokens.shape) != (Bn, self.image_length):
            raise ValueError("img_tokens must have one row per output row: shape %s" % ((Bn, self.image_length),))
        if img_mask is not None:
            want = (Bn, self.image_length)
            if img_tokens is None:
                raise ValueError("img_mask selects positions of img_tokens: pass img_tokens too")
            if not isinstance(img_mask, torch.Tensor) or img_mask.dtype != torch.bool or tuple(img_mask.shape) != want:
                raise ValueError("img_mask must be a bool tensor of shape %s" % (want,))
            if img_tokens.dtype != torch.int64 or tuple(img_tokens.shape) != want:
                raise ValueError("img_tokens must be an int64 tensor of shape %s" % (want,))
            if img_mask.device != dev or img_tokens.device != dev:
                raise ValueError("img_tokens and img_mask must be on the device of text_tokens (%s)" % dev)
            img_tokens, img_mask = img_tokens.contiguous(), img_mask.contiguous()
        if _is_per_row(guidance_scale):
            cfg = scale_rows is not None
        else:
            cfg = guidance_scale is not None and float(guidance_scale) != 1.0
        if cfg:
            if uncond_text_tokens is None:
                uncond_text_tokens = torch.zeros_like(text_tokens)          # all padding -> the per-position pad ids
            text_all = torch.cat([text_tokens, uncond_text_tokens], 0)
            seg_all = torch.cat([seg_tokens, seg_tokens], 0)
        else:
            text_all, seg_all = text_tokens, seg_tokens
        R = text_all.shape[0] * n            # rows [cond: B*n | uncond: B*n]; sample row r belongs to prompt row r // n
        dec = getattr(self, "_sampler", None)
        if (dec is None or dec.rows != R or dec.samples != n or dec.tok.device != dev or not use_graphs
                or dec.version != _param_version(self)):
            dec = _GraphedDecoder(self, R, dev, n)
            if use_graphs:
                self._sampler = dec
        kc, vc = dec.kc, dec.vc
        prefix = text_all.shape[1] + seg_all.shape[1]
        last = self._prefill(self._embed(text_all, seg_all, None), kc, vc)[:, -1].contiguous()
        # expanded BEFORE to_logits: linear_small picks its arithmetic by row count, and the repeated call has R rows here
        logits = self._logits_of(last.repeat_interleave(n, 0) if n > 1 else last)
        toks, kept = [], []
        logprobs = torch.zeros((Bn, self.image_length), dtype=torch.float32, device=dev) if return_logprobs else None

        def uniforms():
            if generator is not None and generator.device.type != dev.type:
                return torch.rand(Bn, generator=generator).to(dev)
            return torch.rand(Bn, device=dev, generator=generator)

        # per-row draw without seeds and without a sampling row: no uniform is read, none is drawn (as a scalar temperature 0)
        u_none = torch.zeros(Bn, dtype=torch.float32, device=dev) if rows is not None and seeds is None and not drawing else None
        for t in range(self.image_length):
            if not cfg:
                mixed = logits
            elif scale_rows is not None:
                mixed = ops.cfg_mix_rows(logits[:Bn], logits[Bn:], scale_rows)
            else:
                mixed = ops.cfg_mix(logits[:Bn], logits[Bn:], guidance_scale)
            if return_logits:
                kept.append(mixed)
            prompt = (img_tokens[:, t], img_mask[:, t]) if img_mask is not None else None
            if img_tokens is not None and prompt is None:
                tok = img_tokens[:, t]
            elif rows is not None:    # per-row controls or seeds: mas_sample_rows, the uniforms of the seeds or of the generator
                u = uniforms() if seeds is None and drawing else u_none
                tok = ops.sample_rows(mixed, *rows, u=u, seeds=seeds, position=t, prompt=prompt,
                                      logp=None if logprobs is None else logprobs[:, t])
            elif not temperature and prompt is None:
                tok = mixed.argmax(-1)
            else:   # prompt, temperature, top-k / top-p filters, softmax and the draw in one kernel; torch only supplies the uniforms
                u = uniforms() if temperature else None
                tok = ops.sample_topk(mixed, float(temperature), top_k, u, top_p=top_p, prompt=prompt,
                                      logp=None if logprobs is None else logprobs[:, t])
            toks.append(tok)
            if t == self.image_length - 1:
                break
            tok_all = torch.cat([tok, tok], 0) if cfg else tok
            logits = (dec.graphed_step if use_graphs else dec.eager_step)(t, tok_all, prefix)
        tokens = torch.stack(toks, 1)
        out = (tokens,) + ((torch.stack(kept, 1),) if return_logits else ()) + ((logprobs,) if return_logprobs else ())
        return out if len(out) > 1 else tokens

    @torch.no_grad()
    def score(self, text_tokens, seg_tokens, img_tokens, guidance_scale=None, uncond_text_tokens=None, num_samples=1):
        """Teacher-forced log-likelihood of given image tokens: fp32 [B,image_length], entry [b, t] = log p(img_t | text, seg,
        img_<t) at temperature 1 with no filters, natural log. With guidance (guidance_scale and uncond_text_tokens as in
        generate) the distribution is softmax(u + s * (c - u)) of the unconditional and conditional streams' logits, the one
        generate draws from at temperature 1 without top_k / top_p. Sum over t to rank candidate images.
        One causal pass over text + seg + image (both streams in one batch with guidance; no dropout, in train mode as in
        eval mode), to_logits on the image_length predicting positions, the guidance mix, then the per-row cross-entropies of
        mas_ce_forward negated. text_tokens [B,text_length], seg_tokens [B,seg_length], img_tokens [B,image_length] (values in
        [0, image_vocab_size)) and uncond_text_tokens [B,text_length]: int64 on the model's device.
        guidance_scale may also give one scale per row (a 1-D tensor on the model's device, or a sequence, of B values, as in
        generate): row b is then the guided log-likelihood at its own scale, bit for bit the row of a call with that scale, so
        candidates can be reranked at several scales in one pass (a row at scale 1 in a guided call: see generate).
        num_samples=n (int >= 1) scores n candidates per prompt, as generate(num_samples=n) draws them: text_tokens,
        seg_tokens and uncond_text_tokens stay per prompt [B,·], img_tokens and the result have B*n rows (row b*n + j is
        candidate j of prompt b), a per-row guidance_scale has B*n values. The result is bit for bit that of
        score(text_tokens.repeat_interleave(n, 0), seg_tokens.repeat_interleave(n, 0), img_tokens, ...) (uncond_text_tokens
        repeated likewise). Where the fused causal-attention core and the fp16 Linear route run (head dim 64 or 128, text +
        seg and image lengths multiples of 128, hidden width a multiple of 128) and the call has at least
        SCORE_SHARED_MIN_ROWS candidate rows (B*n, 2*B*n with guidance), the text + seg prefix is computed once per prompt
        and each candidate's image positions attend to it (mas_attn_causal_prefix_forward): about half the Linear work and
        half the activation memory of the repeated call at the paper's lengths. Elsewhere the prompts are repeated."""
        n = num_samples
        if isinstance(n, bool) or not isinstance(n, int) or n < 1:
            raise ValueError("num_samples must be an int >= 1, got %r" % (num_samples,))
        B = text_tokens.shape[0] if isinstance(text_tokens, torch.Tensor) and text_tokens.dim() == 2 else None
        Bn = None if B is None else B * n
        named = [("text_tokens", text_tokens, self.text_length, B), ("seg_tokens", seg_tokens, self.seg_length, B),
                 ("img_tokens", img_tokens, self.image_length, Bn)]
        if uncond_text_tokens is not None:
            named.append(("uncond_text_tokens", uncond_text_tokens, self.text_length, B))
        dev = self.image_token_embedding.weight.device
        for name, t, length, rows in named:
            if not isinstance(t, torch.Tensor) or B is None or tuple(t.shape) != (rows, length):
                raise ValueError("%s must be a tensor of shape %s" % (name, (rows, length)))
            if t.dtype != torch.int64:
                raise ValueError("%s must be int64, got %s" % (name, t.dtype))
            if t.device != dev:
                raise ValueError("%s must be on the model's device (%s), got %s" % (name, dev, t.device))
        scale_rows = None
        if _is_per_row(guidance_scale):
            scale_h, scale_d = _row_values("guidance_scale", guidance_scale, Bn, dev)
            if not bool(torch.isfinite(scale_h).all()):
                raise ValueError("guidance_scale must be finite in every row, got %s" % scale_h.tolist())
            scale_rows = scale_d if bool((scale_h != 1.0).any()) else None
        V = self.image_token_embedding.num_embeddings
        if bool(((img_tokens < 0) | (img_tokens >= V)).any()):
            raise ValueError("img_tokens must lie in [0, %d)" % V)
        cfg = scale_rows is not None if _is_per_row(guidance_scale) else guidance_scale is not None and float(guidance_scale) != 1.0
        if n > 1 and not self._score_shares_prefix(Bn * (2 if cfg else 1)):
            rep = lambda t: None if t is None else t.repeat_interleave(n, 0)
            return self.score(rep(text_tokens), rep(seg_tokens), img_tokens, guidance_scale, rep(uncond_text_tokens))
        if cfg:
            if uncond_text_tokens is None:
                uncond_text_tokens = torch.zeros_like(text_tokens)          # all padding, as in generate
            text_tokens = torch.cat([text_tokens, uncond_text_tokens], 0)
            seg_tokens, img_all = torch.cat([seg_tokens, seg_tokens], 0), torch.cat([img_tokens, img_tokens], 0)
        else:
            img_all = img_tokens
        L = self.image_length
        if n == 1:
            h = self.transformer.final_ln(self._prefill(self._embed(text_tokens, seg_tokens, img_all)))
            h = h[:, -L - 1:-1].contiguous()                                # forward()'s slice: the predicting positions
        else:
            # prefix rows [cond B | uncond B], candidate rows [cond B*n | uncond B*n]: row r continues prefix row r // n
            ar = torch.arange(L, dtype=torch.long, device=dev)
            ip = self.image_tokens_per_dim
            xs = ops.EmbedFn.apply([(img_all, ar // ip, ar % ip, 0)], L, self.hidden_dim, self.image_token_embedding.weight,
                                   self.image_row_embeddings.weight, self.image_col_embeddings.weight)
            xp, xs = self._prefill_shared(self._embed(text_tokens, seg_tokens, None), xs, n)
            # the predicting positions: the prefix's last one (for image token 0), then image positions 0 .. L-2
            h = self.transformer.final_ln(torch.cat([xp[:, -1:].repeat_interleave(n, 0), xs[:, :-1]], 1))
        logits = self.to_logits[1](self.to_logits[0](h))
        if scale_rows is not None:
            logits = ops.cfg_mix_rows(logits[:Bn], logits[Bn:], scale_rows)
        elif cfg:
            logits = ops.cfg_mix(logits[:Bn], logits[Bn:], guidance_scale)
        return ops.token_logprobs(logits.view(Bn * L, V), img_tokens.reshape(Bn * L)).view(Bn, L)
