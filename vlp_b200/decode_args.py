"""Command-line options of a decode script (the reference's decode_img2txt.py flags) for BertForSeq2SeqDecoder.

    parser = argparse.ArgumentParser()
    decode_args.add_decode_args(parser)                 # --beam_size ... --forbid_duplicate_ngrams ... --sampling_method --topk --topp --seed
    args = decode_args.parse_decode_args(parser)        # argparse's usage error (exit 2) for a combination the decoder refuses
    model = BertForSeq2SeqDecoder.from_pretrained(..., **decode_args.decoder_kwargs(args, tokenizer))

A script that already defines one of these options (decode_img2txt.py has its own --seed, --beam_size, ...) keeps its definition.
"""
import argparse

from . import ops
from .decode import CONSTRAINT_LIMITS, SAMPLING_METHODS, check_decode


def constraint_spec(text):
    """--constraints "dog,dogs|frisbee" -> [["dog", "dogs"], ["frisbee"]]: '|' separates constraints, ',' the alternatives of one;
    argparse.ArgumentTypeError (a usage error) for an empty constraint or alternative, or more than the search takes."""
    cons = [[a.strip() for a in c.split(",")] for c in text.split("|")]
    if any(not a for c in cons for a in c):
        raise argparse.ArgumentTypeError(f"empty constraint or alternative in {text!r} ('|' separates constraints, ',' alternatives)")
    if len(cons) > CONSTRAINT_LIMITS["C"] or any(len(c) > CONSTRAINT_LIMITS["A"] for c in cons):
        raise argparse.ArgumentTypeError(f"at most {CONSTRAINT_LIMITS['C']} constraints of {CONSTRAINT_LIMITS['A']} alternatives, "
                                         f"got {text!r}")
    return cons

_OPTIONS = (
    ("--beam_size", dict(type=int, default=1, help="beam size for beam search; 1 = greedy, and required when sampling")),
    ("--length_penalty", dict(type=float, default=0, help="length penalty for beam search")),
    ("--forbid_duplicate_ngrams", dict(action="store_true", help="never repeat an n-gram (beam search and sampling)")),
    ("--forbid_ignore_word", dict(type=str, default=None, help="'|'-separated words exempt from --forbid_duplicate_ngrams")),
    ("--min_len", dict(type=int, default=None, help="no [SEP] before this many words")),
    ("--ngram_size", dict(type=int, default=3, help="n of --forbid_duplicate_ngrams")),
    ("--sampling_method", dict(type=str, default="beam_search", choices=SAMPLING_METHODS,
                               help="beam_search (greedy at --beam_size 1), or top-k / top-p (nucleus) sampling on the device")),
    ("--topk", dict(type=int, default=1, help=f"--sampling_method topk: sample from the k most likely words, 1 <= k <= {ops.MAX_TOPK}")),
    ("--topp", dict(type=float, default=1.0, help="--sampling_method topp: sample from the smallest set of words whose probability "
                                                  "reaches p, 0 < p <= 1")),
    ("--seed", dict(type=int, default=123, help="random seed (keys the sampling draws)")),
    ("--num_return_sequences", dict(type=int, default=1, help="captions per image: the N best of beam search (N <= --beam_size) or N "
                                                              "top-k / top-p samples, over one K/V cache of the image prefix")),
    ("--num_beam_groups", dict(type=int, default=1, help="diverse beam search: split the --beam_size beams into this many groups, "
                                                         "each penalised for words earlier groups chose in the same step")),
    ("--diversity_penalty", dict(type=float, default=0.0, help="diverse beam search: penalty per earlier group's use of a word, >= 0")),
    ("--constraints", dict(type=constraint_spec, default=None, help="constrained beam search: words or phrases every caption must "
                                                                   "contain, e.g. 'dog,dogs|frisbee' ('|' separates constraints, "
                                                                   "',' the alternatives of one)")),
)


def add_decode_args(parser):
    """Adds every decode option the parser does not define yet; returns the parser."""
    for flag, kw in _OPTIONS:
        try:
            parser.add_argument(flag, **kw)
        except argparse.ArgumentError:
            pass                                               # the script's own definition stays
    return parser


def check_decode_args(args):
    """ValueError for a combination BertForSeq2SeqDecoder refuses (raised before any model is built); --ngram_size is checked with
    --forbid_duplicate_ngrams in every mode, greedy included."""
    check_decode(args.sampling_method, args.topk, args.topp, args.beam_size, args.num_return_sequences, args.forbid_duplicate_ngrams,
                 args.ngram_size, ngram_in_greedy=True, num_beam_groups=args.num_beam_groups, diversity_penalty=args.diversity_penalty,
                 constraints=getattr(args, "constraints", None) is not None)


def parse_decode_args(parser, argv=None):
    """parser.parse_args(argv), then check_decode_args: a refused combination is reported as an argparse usage error (exit 2)."""
    args = parser.parse_args(argv)
    try:
        check_decode_args(args)
    except ValueError as e:
        parser.error(str(e))
    return args


def decoder_kwargs(args, tokenizer=None):
    """BertForSeq2SeqDecoder keyword arguments of the parsed options.  tokenizer (convert_tokens_to_ids) maps --forbid_ignore_word
    to word ids, as decode_img2txt.py does, and tokenizes every --constraints alternative into wordpieces (tokenize, then
    convert_tokens_to_ids); without one both options must be empty."""
    check_decode_args(args)
    ignore = None
    if args.forbid_ignore_word:
        if tokenizer is None:
            raise ValueError("vlp_b200: --forbid_ignore_word needs a tokenizer to map its words to ids")
        ignore = set(tokenizer.convert_tokens_to_ids(args.forbid_ignore_word.split("|")))
    kw = dict(search_beam_size=args.beam_size, length_penalty=args.length_penalty, forbid_duplicate_ngrams=args.forbid_duplicate_ngrams,
              forbid_ignore_set=ignore, ngram_size=args.ngram_size, min_len=args.min_len or 0, sampling_method=args.sampling_method,
              topk=args.topk, topp=args.topp, seed=args.seed)
    if args.num_return_sequences != 1:
        kw["num_return_sequences"] = args.num_return_sequences       # the decoder's default otherwise
    if args.num_beam_groups != 1:
        kw["num_beam_groups"] = args.num_beam_groups
    if args.diversity_penalty != 0:
        kw["diversity_penalty"] = args.diversity_penalty
    if getattr(args, "constraints", None) is not None:
        if tokenizer is None:
            raise ValueError("vlp_b200: --constraints needs a tokenizer to map its words to wordpiece ids")
        kw["constraints"] = [[list(tokenizer.convert_tokens_to_ids(tokenizer.tokenize(a))) for a in c] for c in args.constraints]
    return kw
