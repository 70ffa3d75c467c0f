"""Hyper-parameters of the NMT example.

Parity: the reference's flag set and defaults (`examples/nmt/nmt.py:40-290`
`add_arguments`, `:293-372` `create_hparams`, `:375-474` `extend_hparams`),
the four standard configurations (`examples/nmt/standard_hparams/*.json`, loaded by
`utils/misc_utils.py:maybe_parse_standard_hparams`; here `STANDARD_HPARAMS`) and
`utils/standard_hparams_utils.py:27-104`.

`HParams` is a plain attribute bag with JSON round-trip and
``"a=1,b=foo"`` override strings (the subset of `tf.contrib.training.HParams`
the example uses).
"""
import json
import os

UNK, SOS, EOS = "<unk>", "<s>", "</s>"

# The reference ships four "standard" hyper-parameter files
# (`examples/nmt/standard_hparams/{iwslt15,wmt16,wmt16_gnmt_4_layer,wmt16_gnmt_8_layer}.json`).
# The same settings, written as what they share plus what distinguishes them:
_STD_SHARED = dict(
    batch_size=128, infer_batch_size=32, beam_width=10, num_buckets=5,
    src_max_len=50, tgt_max_len=50, src_max_len_infer=None, tgt_max_len_infer=None,
    optimizer="sgd", learning_rate=1.0, init_weight=0.1, max_gradient_norm=5.0,
    dropout=0.2, forget_bias=1.0, unit_type="lstm", time_major=True,
    sos=SOS, eos=EOS, share_vocab=False, metrics=["bleu"],
    colocate_gradients_with_ops=True, steps_per_external_eval=None)
_WMT = dict(num_units=1024, num_train_steps=340000, decay_scheme="luong10",
            attention="normed_bahdanau", subword_option="bpe")
_GNMT = dict(_WMT, encoder_type="gnmt", attention_architecture="gnmt_v2", residual=True,
             length_penalty_weight=1.0)
STANDARD_HPARAMS = {
    "iwslt15": dict(_STD_SHARED, num_units=512, num_layers=2, num_train_steps=12000,
                    decay_scheme="luong234", encoder_type="bi", attention="scaled_luong",
                    attention_architecture="standard", residual=False, subword_option="",
                    steps_per_stats=100),
    "wmt16": dict(_STD_SHARED, num_layers=4, encoder_type="bi", residual=False,
                  attention_architecture="standard", steps_per_stats=100, **_WMT),
    "wmt16_gnmt_4_layer": dict(_STD_SHARED, num_layers=4, steps_per_stats=100, **_GNMT),
    "wmt16_gnmt_8_layer": dict(_STD_SHARED, num_layers=8, steps_per_stats=50, **_GNMT),
}


class HParams(object):
    def __init__(self, **kw):
        self.__dict__["_keys"] = []
        for k, v in kw.items():
            self.add_hparam(k, v)

    # -- tf.contrib.training.HParams surface ---------------------------------
    def add_hparam(self, name, value):
        if name in self._keys:
            raise ValueError("Hyperparameter name is reserved: %s" % name)
        self._keys.append(name)
        self.__dict__[name] = value

    def set_hparam(self, name, value):
        if name not in self._keys:
            raise KeyError(name)
        self.__dict__[name] = value

    def __setattr__(self, name, value):
        if name not in self._keys:
            self._keys.append(name)
        self.__dict__[name] = value

    def __contains__(self, name):
        return name in self._keys

    def get(self, name, default=None):
        return self.__dict__[name] if name in self._keys else default

    def values(self):
        return {k: self.__dict__[k] for k in self._keys}

    def to_json(self, indent=None):
        return json.dumps(self.values(), indent=indent, sort_keys=True)

    def parse_json(self, text):
        for k, v in (json.loads(text) if isinstance(text, str) else text).items():
            setattr(self, k, v)
        return self

    def parse(self, overrides):
        """``"num_units=32,attention=luong"`` — values are cast to the type of
        the existing value (new names are parsed as int/float/bool/str)."""
        if not overrides:
            return self
        for item in overrides.split(","):
            if not item.strip():
                continue
            k, _, v = item.partition("=")
            k = k.strip()
            setattr(self, k, _cast(v.strip(), self.get(k)))
        return self

    def copy(self):
        return HParams(**json.loads(self.to_json()))

    def __repr__(self):
        return "HParams(%s)" % ", ".join("%s=%r" % (k, self.__dict__[k]) for k in self._keys)


def _cast(text, like):
    if isinstance(like, bool):
        return text.lower() in ("1", "true", "yes")
    if isinstance(like, int):
        return int(text)
    if isinstance(like, float):
        return float(text)
    if isinstance(like, list):
        return [t for t in text.split("|") if t]
    if like is None:
        for fn in (int, float):
            try:
                return fn(text)
            except ValueError:
                pass
        if text.lower() in ("true", "false"):
            return text.lower() == "true"
        if text.lower() in ("none", "null"):
            return None
    return text


def create_standard_hparams():
    """Defaults (`utils/standard_hparams_utils.py:27-104`)."""
    return HParams(
        # data
        src="", tgt="", train_prefix="", dev_prefix="", test_prefix="",
        vocab_prefix="", embed_prefix="", out_dir="",
        # network
        num_units=512, num_layers=2, num_encoder_layers=None, num_decoder_layers=None,
        dropout=0.2, unit_type="lstm", encoder_type="bi", residual=False,
        time_major=True, num_embeddings_partitions=0,
        # attention
        attention="scaled_luong", attention_architecture="standard",
        output_attention=True, pass_hidden_state=True,
        # train
        optimizer="sgd", batch_size=128, init_op="uniform", init_weight=0.1,
        max_gradient_norm=5.0, learning_rate=1.0, warmup_steps=0,
        # True: one global norm over dense variables and embeddings, as the reference
        # clips (`nmt_graph`); False: each embedding's gradient is clipped on its own
        clip_embeddings_jointly=False,
        warmup_scheme="t2t", decay_scheme="luong234",
        colocate_gradients_with_ops=True, num_train_steps=12000,
        # data constraints
        num_buckets=5, max_train=0, src_max_len=50, tgt_max_len=50,
        src_max_len_infer=0, tgt_max_len_infer=0,
        # data format
        sos=SOS, eos=EOS, subword_option="", check_special_token=True,
        # misc
        forget_bias=1.0, num_gpus=1, epoch_step=0, steps_per_stats=100,
        steps_per_external_eval=0, share_vocab=False, metrics=["bleu"],
        log_device_placement=False, random_seed=None, beam_width=0,
        length_penalty_weight=0.0, override_loaded_hparams=True,
        num_keep_ckpts=5, avg_ckpts=False,
        # inference
        inference_indices=None, infer_batch_size=32, sampling_temperature=0.0,
        num_translations_per_input=1,
    )


def standard_hparams_names():
    return sorted(STANDARD_HPARAMS)


def standard_hparams(name_or_path):
    """settings of a bundled standard configuration, or of a JSON file"""
    if name_or_path in STANDARD_HPARAMS:
        return dict(STANDARD_HPARAMS[name_or_path])
    base = os.path.basename(name_or_path)
    if base.endswith(".json") and base[:-5] in STANDARD_HPARAMS and \
            not os.path.exists(name_or_path):
        return dict(STANDARD_HPARAMS[base[:-5]])          # reference-style "…/wmt16.json"
    if os.path.exists(name_or_path):
        with open(name_or_path) as f:
            return json.load(f)
    raise ValueError("unknown standard hparams %r (have: %s)" %
                     (name_or_path, ", ".join(standard_hparams_names())))


def maybe_parse_standard_hparams(hparams, hparams_path):
    """Override `hparams` with a standard configuration (name of a bundled one, or
    the path of a JSON file)."""
    if not hparams_path:
        return hparams
    return hparams.parse_json(standard_hparams(hparams_path))


def load_hparams(model_dir):
    fn = os.path.join(model_dir, "hparams")
    if not os.path.exists(fn):
        return None
    with open(fn) as f:
        try:
            return HParams().parse_json(f.read())
        except ValueError:
            return None


def save_hparams(out_dir, hparams):
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "hparams"), "w") as f:
        f.write(hparams.to_json(indent=1))


def extend_hparams(hparams, src_vocab_size=None, tgt_vocab_size=None):
    """Derived settings and validation (`nmt.py:375-474`): encoder/decoder layer
    counts, residual layer counts, vocabulary sizes, metric bookkeeping."""
    hp = hparams
    # `num_layers` is the legacy spelling; it sets whichever stack depth was not
    # given explicitly (`nmt.py:305-307`)
    hp.num_encoder_layers = hp.get("num_encoder_layers") or hp.num_layers
    hp.num_decoder_layers = hp.get("num_decoder_layers") or hp.num_layers
    if hp.encoder_type == "bi" and hp.num_encoder_layers % 2 != 0:
        raise ValueError("For bi, num_encoder_layers %d should be even" %
                         hp.num_encoder_layers)
    if hp.attention_architecture in ("gnmt", "gnmt_v2") and hp.num_encoder_layers < 2:
        raise ValueError("For gnmt attention architecture, num_encoder_layers %d "
                         "should be >= 2" % hp.num_encoder_layers)
    if hp.subword_option not in ("", "bpe", "spm"):
        raise ValueError("subword option must be either spm, or bpe")
    if hp.beam_width > 0 and hp.sampling_temperature > 0.0:
        raise ValueError("beam search and sampling are mutually exclusive")
    if hp.num_encoder_layers != hp.num_decoder_layers:
        hp.pass_hidden_state = False
    # residual connections start from the second layer (first layer's input is
    # the embedding); GNMT's bidirectional bottom layer is not residual either
    num_enc_res = num_dec_res = 0
    if hp.residual:
        if hp.num_encoder_layers > 1:
            num_enc_res = hp.num_encoder_layers - 1
        if hp.num_decoder_layers > 1:
            num_dec_res = hp.num_decoder_layers - 1
        if hp.encoder_type == "gnmt":
            num_enc_res = hp.num_encoder_layers - 2
            if hp.num_encoder_layers == hp.num_decoder_layers:
                num_dec_res = num_enc_res
    hp.num_encoder_residual_layers = num_enc_res
    hp.num_decoder_residual_layers = num_dec_res
    if src_vocab_size is not None:
        hp.src_vocab_size = int(src_vocab_size)
    if tgt_vocab_size is not None:
        hp.tgt_vocab_size = int(tgt_vocab_size)
    if hp.share_vocab and hp.get("src_vocab_size") and hp.get("tgt_vocab_size"):
        if hp.src_vocab_size != hp.tgt_vocab_size:
            raise ValueError("share_vocab needs equal vocabularies (%d vs %d)" %
                             (hp.src_vocab_size, hp.tgt_vocab_size))
    for m in hp.metrics:
        if "best_" + m not in hp:
            hp.add_hparam("best_" + m, 0.0)
            hp.add_hparam("best_" + m + "_dir", os.path.join(hp.out_dir or "", "best_" + m))
            if hp.avg_ckpts:
                hp.add_hparam("avg_best_" + m, 0.0)
                hp.add_hparam("avg_best_" + m + "_dir",
                              os.path.join(hp.out_dir or "", "avg_best_" + m))
    return hp


def create_hparams(standard=None, overrides=None, **kw):
    """defaults → standard file → keyword arguments → override string."""
    hp = create_standard_hparams()
    maybe_parse_standard_hparams(hp, standard)
    for k, v in kw.items():
        setattr(hp, k, v)
    hp.parse(overrides)
    return hp
