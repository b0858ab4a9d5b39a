"""Options: flag-compatible subset of reference densephrases/options.py (:20-251) for the retrieval hot path --
every flag `eval_phrase_retrieval.py`, `DensePhrases.__init__` (model.py:30-43) and the Makefile eval targets
(Makefile:169-181) pass is accepted with the reference's default; training/dump-only flags are accepted and ignored."""
import argparse
import os


class Options(object):
    def __init__(self):
        self.parser = argparse.ArgumentParser()
        self.initialized = False
        self._add_common()

    def _add_common(self):
        p = self.parser
        p.add_argument("--seed", type=int, default=42)
        p.add_argument("--draft", action="store_true")
        p.add_argument("--verbose_logging", action="store_true")
        p.add_argument("--fp16", action="store_true")
        p.add_argument("--fp16_opt_level", type=str, default="O1")
        p.add_argument("--local_rank", type=int, default=-1)

    def add_model_options(self):
        p = self.parser
        p.add_argument("--model_type", type=str, default='bert')
        p.add_argument("--pretrained_name_or_path", type=str, default='SpanBERT/spanbert-base-cased')
        p.add_argument("--config_name", type=str, default="")
        p.add_argument("--tokenizer_name", type=str, default="")
        p.add_argument("--load_dir", type=str, default="")
        p.add_argument("--output_dir", type=str, default=None)
        p.add_argument("--max_seq_length", type=int, default=384)
        p.add_argument("--doc_stride", type=int, default=128)
        p.add_argument("--max_query_length", type=int, default=64)
        p.add_argument("--max_answer_length", type=int, default=10)
        p.add_argument("--do_lower_case", action="store_true")

    def add_index_options(self):
        p = self.parser
        p.add_argument('--stage', type=str)
        p.add_argument('--dump_dir', type=str)
        p.add_argument('--offset', type=int, default=0)
        p.add_argument('--phrase_dir', default='phrase')
        p.add_argument('--index_name', default='start/256_flat_SQ4')
        p.add_argument('--index_path', default='index.faiss')
        p.add_argument('--idx2id_path', default='idx2id.hdf5')
        p.add_argument('--num_clusters', type=int, default=16384)
        p.add_argument('--fine_quant', default='SQ4')
        p.add_argument('--cuda', action='store_true', default=False)
        p.add_argument('--replace', action='store_true', default=False)
        # build-side flags of build_phrase_index.py (options.py:57-68): declared for flag compatibility, unused on the serving path
        for name in ('add_all', 'hnsw', 'first_passage'):
            p.add_argument(f'--{name}', action='store_true', default=False)
        p.add_argument('--norm_th', type=float, default=999)
        p.add_argument('--doc_sample_ratio', type=float, default=0.2)
        p.add_argument('--vec_sample_ratio', type=float, default=0.2)
        p.add_argument('--num_docs_per_add', type=int, default=2000)
        p.add_argument('--index_filter', type=float, default=-1e8)
        for name, default in (('quantizer_path', 'quantizer.faiss'), ('trained_index_path', 'trained.faiss'), ('inv_path', 'merged.invdata'),
                              ('subindex_name', 'index'), ('dump_paths', None)):
            p.add_argument(f'--{name}', default=default)

    def add_retrieval_options(self):
        p = self.parser
        p.add_argument('--run_mode', default='eval')
        p.add_argument('--top_k', type=int, default=10)
        p.add_argument('--nprobe', type=int, default=256)
        p.add_argument('--aggregate', action='store_true', default=False)
        p.add_argument('--agg_strat', type=str, default='opt1')
        p.add_argument('--dev_path', default='open-qa/nq-open/dev_preprocessed.json')
        p.add_argument('--test_path', default='open-qa/nq-open/test_preprocessed.json')
        p.add_argument('--candidate_path', default=None)
        p.add_argument('--regex', action='store_true', default=False)
        p.add_argument('--eval_batch_size', type=int, default=64)
        p.add_argument('--save_pred', action='store_true', default=False)
        p.add_argument('--eval_psg', action='store_true', default=False)
        p.add_argument('--psg_top_k', type=int, default=100)
        p.add_argument('--max_psg_len', type=int, default=999999999)
        p.add_argument('--mark_phrase', action='store_true', default=False)
        p.add_argument('--return_sent', action='store_true', default=False)
        p.add_argument('--sent_window', type=int, default=0)
        p.add_argument('--is_kilt', action='store_true', default=False)
        p.add_argument('--kilt_gold_path', default='kilt/trex/trex-dev-kilt.jsonl')
        p.add_argument('--title2wikiid_path', default='wikidump/title2wikiid.json')

    def add_data_options(self):
        p = self.parser
        p.add_argument("--data_dir", type=str, default=None)
        p.add_argument("--cache_dir", type=str, default="")
        p.add_argument("--threads", type=int, default=20)
        p.add_argument("--truecase_path", type=str, default='truecase/english_with_questions.dist')
        p.add_argument("--truecase", action="store_true")

    # accepted for command-line compatibility; nothing on the retrieval path reads them
    def add_rc_options(self):
        p = self.parser
        for name in ('lambda_kl', 'lambda_neg', 'lambda_flt'):
            p.add_argument(f'--{name}', default=0.0, type=float)
        p.add_argument('--dense_offset', type=float, default=-2)
        p.add_argument('--dense_scale', type=float, default=20)

    def add_qsft_options(self):
        p = self.parser
        p.add_argument('--train_path', default=None)
        p.add_argument('--label_strat', default='phrase', type=str)

    def add_demo_options(self):
        p = self.parser
        p.add_argument('--base_ip', default='http://127.0.0.1')
        p.add_argument('--query_port', type=str, default='-1')
        p.add_argument('--index_port', type=str, default='-1')

    def initialize(self):
        self.initialized = True

    def parse(self, argv=None):
        opt, _ = self.parser.parse_known_args(argv) if argv is not None else self.parser.parse_known_args()
        if getattr(opt, 'dump_dir', None) is not None and os.environ.get('SAVE_DIR') and not os.path.isabs(opt.dump_dir):
            opt.dump_dir = os.path.join(os.environ['SAVE_DIR'], opt.dump_dir)
        self.opt = opt
        return opt
