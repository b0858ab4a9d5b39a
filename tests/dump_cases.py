"""Shared inputs of the phrase-dump tests and their golden generator (tests/golden/make_dump_golden.py): the synthetic documents,
the tokenizer's vocabulary, the dump settings of each case, and the phrase tower's fp32 outputs regenerated from a seed."""
import numpy as np

from densephrases_b200.tokenization import WordPieceTokenizer

WORDS = ['Paris', 'river', 'Seine', 'flows', 'through', 'the', 'city', "France's", 'capital', 'since', '1850,', 'bridges', 'cross',
         'it', 'many', 'times', 'and', 'boats', 'carry', 'tourists', 'unbelievably', 'slowly', '(north)', 'St.', 'Louis', 'a']
QUIET_DOC = 2          # every logit of this document is -5, and its first row's filter_start -1e7: filtered out at -2.0 and 0.1

# name, S, doc_stride, append_title, max_answer_length, thresholds, dense_offset, dense_scale, output seed
CASES = [
    ('title_s64_d20_L10', 64, 20, True, 10, [-1e8, -2.0, 0.1], -2.0, 20.0, 11),
    ('notitle_s64_d50_L64', 64, 50, False, 64, [-2.0, 0.1], -2.0, 4.0, 12),
    ('title_s64_d50_L1', 64, 50, True, 1, [0.1], -2.0, 20.0, 13),
]
FILTER_ONLY_CASE = 'title_s64_d20_L10'


def tokenizer():
    return WordPieceTokenizer.from_pretrained_or_synthetic(None, extra_words=WORDS[:20])


def documents(seed=5):
    """SQuAD-style `data`: multi-paragraph documents, paragraphs longer than one window, a skipped is_paragraph: false paragraph,
    a list title with underscores, non-breaking spaces, and the quiet document."""
    rng = np.random.default_rng(seed)
    text = lambda n: ' '.join(WORDS[i] for i in rng.integers(0, len(WORDS), n))      # noqa: E731
    return [
        {'title': 'River_Seine', 'paragraphs': [{'context': text(30)}, {'context': text(70)}, {'context': text(12)}]},
        {'title': ['Paris  capital', 'other'], 'paragraphs': [{'context': text(20), 'is_paragraph': False},
                                                              {'context': text(25).replace(' ', '\xa0', 3)}, {'context': text(90)}]},
        {'title': 'Quiet', 'paragraphs': [{'context': text(40)}, {'context': text(8)}]},
        {'title': 'Boats of St. Louis and the unbelievably slow tourists of France', 'paragraphs': [{'context': text(15)}]},
        {'title': '', 'paragraphs': [{'context': text(5)}, {'context': text(60), 'is_paragraph': True}]},
    ]


def phrase_outputs(features, S, seed, row_lo):
    """fp32 start [F,S,768] and filter logits [F,S,2] for the features: normal values mixed with odd multiples of 1/8 around -2
    (exactly .5 after (x + 2) * 4, and past the int8 clip); logits on a quarter grid with exact fp32(0.1) and -2.0 entries."""
    rng = np.random.default_rng(seed)
    F = len(features)
    start = (rng.standard_normal((F, S, 768)) * 3).astype(np.float32)
    grid = (-2.0 + (rng.integers(-600, 600, (F, S, 768)) * 2 + 1) / 8.0).astype(np.float32)
    start = np.where(rng.random((F, S, 768)) < 0.25, grid, start)
    logits = (np.round(rng.normal(size=(F, S, 2)) * 8.0) / 4.0).astype(np.float32)
    u = rng.random((F, S, 2))
    logits[u < 0.08] = np.float32(0.1)
    logits[(u >= 0.08) & (u < 0.14)] = np.float32(-2.0)
    first = True
    for i, f in enumerate(features):
        if f.doc_idx == QUIET_DOC:
            logits[i] = -5.0
            if first:
                logits[i, row_lo[i], 0] = -1e7
                first = False
    return start, logits
