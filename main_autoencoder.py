#!/usr/bin/env python
"""CLI with the reference's flag surface (reference main_autoencoder.py:23-111) driving the H100 DenoisingAutoencoder.

    python main_autoencoder.py --model_name uci --verbose --encode_full [--data_path datasets/uci_news.snappy.parquet]
    python main_autoencoder.py --model_name syn --synthetic 100000 --num_epochs 2 --batch_size 800 --verbose

Same flag names, defaults, asserts and `.env` override as the reference (python-dotenv; the two env typos at
main_autoencoder.py:79-80 are fixed and `adam` is accepted, SURVEY appendix A).  Data preparation follows
main_autoencoder.py:177-238 (CountVectorizer -> binary / tf-idf CSR, factorised labels).  The evaluation tail (:307-360) runs on
the GPU as numbers, not pictures: pairwise similarity of the inputs and of the embeddings, related-vs-unrelated AUROC + box
statistics (one JSON per reference plot file name under <plot_dir>) and the most-similar-article lookup; drawing with matplotlib
is not reproduced.
"""
import argparse
import os
from pathlib import Path

import numpy as np

_script_path = Path(os.path.dirname(os.path.realpath(__file__)))


def _bool_flag(ap, name, default, help_):
    ap.add_argument('--' + name, dest=name, action='store_true', default=default, help=help_)
    ap.add_argument('--no' + name, dest=name, action='store_false')


def build_parser():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    _bool_flag(ap, 'verbose', False, 'Level of verbosity. 0 - silent, 1 - print log')
    ap.add_argument('--verbose_step', type=int, default=5)
    _bool_flag(ap, 'encode_full', False, 'Whether to encode and store the full data set')
    _bool_flag(ap, 'validation', False, 'Whether to use a validation set and print validation loss')
    ap.add_argument('--input_format', default='binary', help='["binary", "tfidf"]')
    ap.add_argument('--label', default='category_publish_name', help='["category_publish_name", "story"]')
    _bool_flag(ap, 'save_tsv', False, 'Whether to save data in tsv format')
    ap.add_argument('--train_row', type=int, default=8000)
    ap.add_argument('--validate_row', type=int, default=2000)
    _bool_flag(ap, 'restore_previous_data', False, 'restore previous data corresponding to model name')
    ap.add_argument('--min_df', type=float, default=0.0)
    ap.add_argument('--max_df', type=float, default=0.99)
    ap.add_argument('--max_features', type=int, default=10000)
    ap.add_argument('--model_name', default='')
    _bool_flag(ap, 'restore_previous_model', False, 'restore previous model corresponding to model name')
    ap.add_argument('--seed', type=int, default=-1)
    ap.add_argument('--compress_factor', type=int, default=20)
    ap.add_argument('--corr_type', default='masking', help='["none", "masking", "salt_and_pepper", "decay"]')
    ap.add_argument('--corr_frac', type=float, default=0.3)
    ap.add_argument('--xavier_init', type=int, default=1)
    ap.add_argument('--enc_act_func', default='sigmoid')
    ap.add_argument('--dec_act_func', default='sigmoid')
    ap.add_argument('--main_dir', default='')
    ap.add_argument('--loss_func', default='cross_entropy')
    ap.add_argument('--opt', default='gradient_descent', help='["gradient_descent", "ada_grad", "momentum", "adam"]')
    ap.add_argument('--learning_rate', type=float, default=0.1)
    ap.add_argument('--momentum', type=float, default=0.5)
    ap.add_argument('--num_epochs', type=int, default=50)
    ap.add_argument('--batch_size', type=float, default=0.1)
    ap.add_argument('--alpha', type=float, default=1.0)
    ap.add_argument('--triplet_strategy', default='batch_all')
    # additive
    ap.add_argument('--data_path', default='datasets/uci_news.snappy.parquet')
    ap.add_argument('--synthetic', type=int, default=0, help='train on N synthetic articles instead of reading --data_path')
    ap.add_argument('--rng_mode', default='device', choices=['numpy', 'device'],
                    help="'device': Philox masking + device permutation (default); 'numpy': the reference's host NumPy RNG stream")
    ap.add_argument('--top_k', type=int, default=0,
                    help='K > 0: after transform, save the K most similar training articles of every training and every validation '
                         'article (K <= 32, or K <= 1024 with --long_lists) and report the share that shares the label; 0 = off')
    ap.add_argument('--long_lists', action='store_true', default=False,
                    help='let --top_k K go up to 1024 (the long-list stages of helpers.top_k_similar / recommend) for the article '
                         'lists, the user lists and --top_k_dedup; not with --top_k_input, whose sparse ranking stops at 32')
    ap.add_argument('--top_k_input', action='store_true', default=False,
                    help='with --top_k K: also rank by the input vectors (cosine for binary, linear kernel for tf-idf), save '
                         'article_top_k_input_{index,score}[_validate].npy and report their label precision next to the embedding\'s')
    ap.add_argument('--top_k_dedup', type=float, default=0.0,
                    help='with --top_k K: T > 0 groups the training articles whose embedding cosine similarity is >= T (near-duplicates, '
                         'helpers.similar_pairs + duplicate_groups) and saves K-best lists with at most one article per group as '
                         'article_top_k_dedup_{index,score}[_validate].npy (and user_top_k_dedup_{index,score}.npy with '
                         '--user_histories, read groups excluded); their label precision (and hit rate / recall) is reported next to '
                         'the plain lists\'; 0 = off')
    ap.add_argument('--dedup_threshold', type=float, default=0.0,
                    help='T > 0: after transform, list every pair of training articles whose embedding cosine similarity is >= T '
                         '(near-duplicates) and every (validation, training) pair, save them with their duplicate groups as '
                         'article_duplicates[_validate].npz (i, j, score, group) and report the pair and group counts and the '
                         'precision / recall against --label; 0 = off')
    ap.add_argument('--dedup_input', action='store_true', default=False,
                    help='with --dedup_threshold T: the same on the input vectors (cosine for binary, linear kernel for tf-idf), saved '
                         'as article_duplicates_input[_validate].npz and reported next to the embedding\'s numbers')
    ap.add_argument('--eval_all_rows', action='store_true', default=False,
                    help='evaluate sets above 20 000 rows instead of skipping them: AUROC and box statistics from score histograms '
                         '(helpers.similarity_auroc, reported with their error bound) and the nearest article through top_k_similar')
    ap.add_argument('--mining_block_rows', type=int, default=0,
                    help='R > 0 (a multiple of 128 up to 32768): batch_all / batch_hard mine the similarity matrix R rows at a time '
                         '(12 R B bytes instead of 12 B^2), which trains batches above 32 768 rows; 0 = off')
    ap.add_argument('--deterministic', action='store_true', default=False,
                    help='add every floating-point sum of the training step in a fixed order, so that a rerun with the same --seed (>= 0) '
                         'and data gives bit-identical parameters, losses and embeddings on the same GPU model (slower; default: off, '
                         'or the environment variable DAE_DETERMINISTIC=1); this covers the DAE step only, see --user_deterministic for the '
                         'user encoder')
    ap.add_argument('--user_histories', default='',
                    help='with --top_k K: a scipy.sparse.save_npz matrix [users x training articles] of reading histories (values: '
                         'weights); after transform, recommend the K best unread training articles to every user (helpers.recommend) '
                         'and save user_top_k_{index,score}.npy')
    ap.add_argument('--user_sequences', default='',
                    help='with --top_k K: an .npz with indptr [users + 1] and items (training article rows in reading order), '
                         'optionally targets [users] (the next read, -1 = none); train a GRU user encoder (user_model.UserGRU) on '
                         'the training embeddings, save user_gru.npz and user_gru_top_k_{index,score}.npy; with targets report '
                         'user_gru_hit_rate / user_gru_recall next to the mean profile\'s for the same reads')
    ap.add_argument('--user_epochs', type=int, default=5, help='with --user_sequences: training epochs of the GRU user encoder')
    ap.add_argument('--user_cell', default='gru', choices=['gru', 'lstm', 'attention'],
                    help='with --user_sequences: the user encoder, user_model.UserGRU (gru, the default), user_model.UserLSTM (lstm) '
                         'or user_model.UserAttention (attention: NRMS\'s causal self-attention and additive pooling); the files '
                         'and keys say user_<cell> in place of user_gru')
    ap.add_argument('--user_heads', type=int, default=None,
                    help='with --user_cell attention: attention heads, a divisor of the embedding width with at most 128 '
                         'columns per head (default: its largest divisor <= 20)')
    ap.add_argument('--user_attention_dim', type=int, default=None,
                    help='with --user_cell attention: width of the additive pooling layer (default 200)')
    ap.add_argument('--user_long_term', action='store_true', default=False,
                    help='with --user_sequences and --user_cell gru or lstm: learn a long-term vector per user (one row per sequence '
                         'row) and start each user\'s window of recent reads from it (LSTUR-ini, DESIGN 4.18)')
    ap.add_argument('--user_long_term_mask', type=float, default=None,
                    help='with --user_long_term: the probability that a training batch user starts from 0 instead (default 0.5)')
    ap.add_argument('--user_long_term_lr', type=float, default=None,
                    help='with --user_long_term: the learning rate of the long-term vectors (default '
                         'user_model.LONG_TERM_LEARNING_RATE)')
    ap.add_argument('--user_fine_tune_articles', action='store_true', default=False,
                    help='with --user_sequences: train the DAE encoder (W, bh) together with the user encoder on its loss '
                         '(user_model.ArticleEncoder, inputs scaled by 1 - corr_frac); save user_<cell>_article_encoder.npz and '
                         'article_encoded_fine_tuned.npy, and score the user encoder with the fine-tuned vectors (the mean profile '
                         'keeps the DAE\'s)')
    ap.add_argument('--user_deterministic', action='store_true', default=False,
                    help='with --user_sequences: train the user encoder (and with --user_fine_tune_articles the article encoder) in '
                         'its deterministic mode, so that a rerun on the same embeddings gives bit-identical parameters and losses on '
                         'the same GPU model (DESIGN 4.21); for a whole run to repeat, also pass --deterministic and --seed >= 0')
    ap.add_argument('--user_article_lr', type=float, default=None,
                    help='with --user_fine_tune_articles: the article encoder\'s learning rate (default '
                         'user_model.ARTICLE_LEARNING_RATE)')
    ap.add_argument('--user_impressions', default='',
                    help='with --user_sequences: an .npz impression log (user, time, indptr, items, clicked; see '
                         'user_model.check_impressions) to train the GRU on instead of random negatives')
    ap.add_argument('--user_impression_loss', default=None, choices=['pairwise', 'softmax'],
                    help='with --user_impressions: the impression loss, pairwise (every click against every non-click; the '
                         'default) or softmax (each click against --user_negatives non-clicks of its impression under a softmax '
                         'cross-entropy, as MIND\'s trainers do)')
    ap.add_argument('--user_negatives', type=int, default=None,
                    help='with --user_impressions: K, the non-clicks drawn per click by --user_impression_loss softmax, '
                         '0 <= K <= 32 (default 4; 0 = every non-click)')
    ap.add_argument('--user_test_impressions', default='',
                    help='with --user_sequences: an .npz impression log to score; report the AUC, MRR, nDCG@5 and nDCG@10 of the '
                         'GRU states (user_gru_imp_*) and of the mean profile of the same reads (user_mean_imp_*)')
    ap.add_argument('--user_top_k_input', action='store_true', default=False,
                    help='with --top_k K (1..32) and --user_histories or --user_sequences: also recommend from the bag-of-words '
                         'profiles of the same reads (helpers.recommend_sparse; cosine for binary, linear kernel for tf-idf, as '
                         '--top_k_input); with --user_histories save user_top_k_input_{index,score}.npy and report '
                         'user_input_hit_rate / user_input_recall, with --user_sequences report user_input_seq_hit_rate / '
                         '_recall and, with --user_test_impressions, user_input_imp_* next to the user encoder\'s and the mean '
                         'profile\'s')
    ap.add_argument('--user_targets', default='',
                    help='with --user_histories: a save_npz matrix of the same shape holding held-out reads; report the hit rate '
                         'and recall of the recommendations against them (user_hit_rate, user_recall)')
    return ap


def apply_env_overrides(flags):
    """Same-named environment variables (loaded from .env) override the flags (reference main_autoencoder.py:13-17,36-92)."""
    dot_env_path = _script_path / '.env'
    if dot_env_path.exists():
        try:
            import dotenv
            print('.env found, will override all flags using values in .env')
            dotenv.load_dotenv(dot_env_path)
        except ImportError:
            pass
    for k, cast in _ENV_OVERRIDES.items():   # the reference's fixed list (main_autoencoder.py:75-92), with the right keys for corr_*
        if k in os.environ and hasattr(flags, k):
            setattr(flags, k, cast(os.environ[k]))
    return flags


def _env_bool(raw):
    """The reference sets a boolean flag to True when the variable merely exists; here '0' / 'false' / 'no' / '' mean False."""
    return str(raw).strip().lower() not in ('', '0', 'false', 'no', 'off')


_ENV_OVERRIDES = {'model_name': str, 'restore_previous_model': _env_bool, 'seed': int, 'compress_factor': int, 'corr_type': str,
                  'corr_frac': float, 'xavier_init': int, 'enc_act_func': str, 'dec_act_func': str, 'main_dir': str, 'loss_func': str,
                  'opt': str, 'learning_rate': float, 'momentum': float, 'num_epochs': int, 'batch_size': float, 'alpha': float,
                  'triplet_strategy': str}


def check_flags(F):
    assert 0. <= F.min_df <= 1.
    assert 0. <= F.max_df <= 1.
    assert F.max_features >= 1
    assert F.enc_act_func in ['sigmoid', 'tanh']
    assert F.dec_act_func in ['sigmoid', 'tanh', 'none']
    assert F.corr_type in ['masking', 'salt_and_pepper', 'decay', 'none']
    assert 0. <= F.corr_frac <= 1.
    assert F.loss_func in ['cross_entropy', 'mean_squared', 'cosine_proximity']
    assert F.opt in ['gradient_descent', 'ada_grad', 'momentum', 'adam']
    assert F.verbose_step > 0
    assert F.triplet_strategy in ['batch_all', 'batch_hard', 'none']
    assert F.input_format in ['binary', 'tfidf']
    assert F.label in ['category_publish_name', 'story']
    assert 0 <= F.top_k <= (1024 if F.long_lists else 32), '--top_k %d: K <= 32, or K <= 1024 with --long_lists' % F.top_k
    if F.top_k_input and F.top_k > 32:
        raise ValueError('--top_k_input ranks the sparse input vectors, at most 32 results per article: --top_k %d needs K <= 32'
                         % F.top_k)
    assert not F.top_k_input or F.top_k > 0, '--top_k_input needs --top_k K > 0'
    assert F.top_k_dedup >= 0.0
    assert not F.top_k_dedup or F.top_k > 0, '--top_k_dedup needs --top_k K > 0'
    assert F.dedup_threshold >= 0.0
    assert not F.dedup_input or F.dedup_threshold > 0, '--dedup_input needs --dedup_threshold T > 0'
    assert not F.user_histories or F.top_k > 0, '--user_histories needs --top_k K > 0'
    assert not F.user_histories or os.path.isfile(F.user_histories), '--user_histories %s: no such file' % F.user_histories
    assert not F.user_sequences or F.top_k > 0, '--user_sequences needs --top_k K > 0'
    assert not F.user_sequences or os.path.isfile(F.user_sequences), '--user_sequences %s: no such file' % F.user_sequences
    assert F.user_epochs >= 0, '--user_epochs must be >= 0'
    for flag, path in (('--user_impressions', F.user_impressions), ('--user_test_impressions', F.user_test_impressions)):
        assert not path or F.user_sequences, '%s needs --user_sequences' % flag
        assert not path or os.path.isfile(path), '%s %s: no such file' % (flag, path)
    for flag, v in (('--user_impression_loss', F.user_impression_loss), ('--user_negatives', F.user_negatives)):
        assert v is None or F.user_impressions, '%s needs --user_impressions' % flag
    F.user_impression_loss = F.user_impression_loss or 'pairwise'
    for flag, v in (('--user_heads', F.user_heads), ('--user_attention_dim', F.user_attention_dim)):
        assert v is None or F.user_cell == 'attention', '%s needs --user_cell attention' % flag
    assert F.user_heads is None or F.user_heads >= 1, '--user_heads must be >= 1'
    assert not F.user_long_term or F.user_sequences, '--user_long_term needs --user_sequences'
    assert not F.user_long_term or F.user_cell in ('gru', 'lstm'), '--user_long_term needs --user_cell gru or lstm'
    for flag, v in (('--user_long_term_mask', F.user_long_term_mask), ('--user_long_term_lr', F.user_long_term_lr)):
        assert v is None or F.user_long_term, '%s needs --user_long_term' % flag
    F.user_long_term_mask = 0.5 if F.user_long_term_mask is None else F.user_long_term_mask
    assert 0.0 <= F.user_long_term_mask <= 1.0, '--user_long_term_mask must lie in [0, 1]'
    assert F.user_long_term_lr is None or F.user_long_term_lr > 0, '--user_long_term_lr must be > 0'
    assert not F.user_fine_tune_articles or F.user_sequences, '--user_fine_tune_articles needs --user_sequences'
    assert F.user_article_lr is None or F.user_fine_tune_articles, '--user_article_lr needs --user_fine_tune_articles'
    assert not F.user_deterministic or F.user_sequences, '--user_deterministic needs --user_sequences'
    assert F.user_article_lr is None or F.user_article_lr >= 0, '--user_article_lr must be >= 0'
    F.user_attention_dim = 200 if F.user_attention_dim is None else F.user_attention_dim
    assert F.user_attention_dim >= 1, '--user_attention_dim must be >= 1'
    F.user_negatives = 4 if F.user_negatives is None else F.user_negatives
    assert 0 <= F.user_negatives <= 32, '--user_negatives %d: 0 <= K <= 32' % F.user_negatives
    assert not F.user_targets or F.user_histories, '--user_targets needs --user_histories'
    assert not F.user_targets or os.path.isfile(F.user_targets), '--user_targets %s: no such file' % F.user_targets
    assert not F.user_top_k_input or 1 <= F.top_k <= 32, '--user_top_k_input needs --top_k K in 1..32'
    assert not F.user_top_k_input or F.user_histories or F.user_sequences, \
        '--user_top_k_input needs --user_histories or --user_sequences'
    if F.input_format == 'tfidf':
        assert F.loss_func in ['mean_squared', 'cosine_proximity']
    if F.main_dir == '':
        F.main_dir = F.model_name
    return F


_LABELS = ('category_publish_name', 'story')
_TSV_LABEL_COLUMNS = ['label_story', 'label_category_publish_name', 'title', 'story', 'category_publish_name']


def prepare_uci(F, model=None):
    """main_autoencoder.py:177-244 with pandas >= 2 fixes (sort by the article_id column, no DataFrame.append): vectorise the
    newest train_row + validate_row articles and, when a model is given, write the data_dir cache the reference writes
    (same file names and formats) so that --restore_previous_data finds it."""
    import joblib
    import pandas as pd
    from sklearn.feature_extraction.text import CountVectorizer, TfidfTransformer
    from dae_rnn_news_recommendation_b200.io_formats import save_file
    df = pd.read_parquet(F.data_path)
    if 'article_id' in df.columns:
        df = df.set_index('article_id', drop=False)
        df.index.name = None
    df = df.sort_index(ascending=False)
    df['label_story'] = pd.factorize(df.story)[0]
    cat = df.category_publish_name.apply(lambda s: s.lstrip('即時') if isinstance(s, str) else s)
    df['label_category_publish_name'] = pd.factorize(cat)[0]
    if F.triplet_strategy != 'none':
        # rows without the selected label cannot be mined (reference main_autoencoder.py:181-201 keeps label_<label>_valid == 1):
        # pd.factorize gives them -1, which would otherwise act as one large shared class
        df = df.loc[df['label_' + F.label] >= 0]
    n_tr, n_va = F.train_row, F.validate_row
    df = df.iloc[0:n_tr + n_va].sample(frac=1)
    df = df.sort_values('article_id') if 'article_id' in df.columns else df.sort_index()
    def df_bound(v):   # sklearn >= 1.2 validates: a proportion is a float in [0, 1], a document count an int >= 1
        return float(v) if v <= 1 else int(v)
    cv = CountVectorizer(stop_words='english', min_df=df_bound(F.min_df), max_df=df_bound(F.max_df), max_features=F.max_features,
                         binary=False)
    X = cv.fit_transform(df.main_content[0:n_tr])
    Xv = cv.transform(df.main_content[n_tr:n_tr + n_va])
    tf = TfidfTransformer()
    Xt, Xtv = tf.fit_transform(X), tf.transform(Xv)
    d = {'articles': df.iloc[0:n_tr], 'articles_validate': df.iloc[n_tr:n_tr + n_va], 'tfidf': (Xt, Xtv),
         'count_vectorizer': cv, 'tfidf_transformer': tf}
    for lab in _LABELS:
        d['label_' + lab] = (df['label_' + lab][0:n_tr], df['label_' + lab][n_tr:n_tr + n_va])
    if model is not None:
        dd = model.data_dir
        save_file(d['articles'], dd + 'article.snappy.parquet')
        save_file(d['articles_validate'], dd + 'article_validate.snappy.parquet')
        for lab in _LABELS:
            save_file(d['label_' + lab][0], dd + 'article_label_%s.pkl' % lab)
            save_file(d['label_' + lab][1], dd + 'article_label_%s_validate.pkl' % lab)
        save_file(X, dd + 'article_count_vectorized.npz')
        save_file(Xv, dd + 'article_count_vectorized_validate.npz')
    X.data = np.ones(len(X.data), dtype=X.data.dtype)      # binary bag of words (main_autoencoder.py:234-235)
    Xv.data = np.ones(len(Xv.data), dtype=Xv.data.dtype)
    d['binary'] = (X, Xv)
    if model is not None:
        save_file(X, dd + 'article_binary_count_vectorized.npz')
        save_file(Xv, dd + 'article_binary_count_vectorized_validate.npz')
        save_file(Xt, dd + 'article_tfidf_vectorized.npz')
        save_file(Xtv, dd + 'article_tfidf_vectorized_validate.npz')
        joblib.dump(cv, dd + 'count_vectorizer.joblib')
        joblib.dump(tf, dd + 'tfidf_transformer.joblib')
    return d


def restore_uci(model):
    """--restore_previous_data (main_autoencoder.py:161-175): read back the cache of an earlier run with the same model name."""
    import joblib
    from dae_rnn_news_recommendation_b200.io_formats import read_file
    dd = model.data_dir
    d = {'articles': read_file(dd + 'article.snappy.parquet'), 'articles_validate': read_file(dd + 'article_validate.snappy.parquet'),
         'binary': (read_file(dd + 'article_binary_count_vectorized.npz'), read_file(dd + 'article_binary_count_vectorized_validate.npz')),
         'tfidf': (read_file(dd + 'article_tfidf_vectorized.npz'), read_file(dd + 'article_tfidf_vectorized_validate.npz')),
         'count_vectorizer': joblib.load(dd + 'count_vectorizer.joblib'), 'tfidf_transformer': joblib.load(dd + 'tfidf_transformer.joblib')}
    for lab in _LABELS:
        d['label_' + lab] = (read_file(dd + 'article_label_%s.pkl' % lab, data_type='pandas_series'),
                             read_file(dd + 'article_label_%s_validate.pkl' % lab, data_type='pandas_series'))
    return d


def save_tsv(model, d, enc, enc_v):
    """--save_tsv (main_autoencoder.py:292-301): the projector-ready TSV set under tsv_dir."""
    from dae_rnn_news_recommendation_b200.io_formats import save_file
    td = model.tsv_dir
    if d is not None:
        for name in ('tfidf', 'binary'):
            stem = 'article_tfidf_vectorized' if name == 'tfidf' else 'article_binary_count_vectorized'
            save_file(d[name][0], td + stem + '.tsv')
            save_file(d[name][1], td + stem + '_validate.tsv')
        cols = [c for c in _TSV_LABEL_COLUMNS if c in d['articles'].columns]
        save_file(d['articles'][cols], td + 'article_label.tsv')
        save_file(d['articles_validate'][cols], td + 'article_label_validate.tsv')
    save_file(np.asarray(enc), td + 'article_encoded.tsv')
    save_file(np.asarray(enc_v), td + 'article_encoded_validate.tsv')


def prepare_synthetic(F):
    from dae_rnn_news_recommendation_b200.synth import make_sparse, make_labels
    n = F.synthetic
    X = make_sparse(n, F.max_features, 100, 'binary' if F.input_format == 'binary' else 'tfidf', seed=max(F.seed, 0))
    lab = make_labels(n, 4, seed=max(F.seed, 0))
    nv = min(F.validate_row, n // 5)
    return X[:n - nv], X[n - nv:], lab[:n - nv], lab[n - nv:]


def evaluate(F, model, trX, vlX, trL, vlL, enc, enc_v, max_rows=20000):
    """Reference main_autoencoder.py:307-360: cosine similarity of the input space and of the embeddings, the related / unrelated
    comparison for the label in use, and the nearest article of the first rows.  N x N lives on the GPU only; sets larger than
    `max_rows` (the reference runs 8000 / 2000 rows) are skipped -- or, with --eval_all_rows, evaluated without the N x N matrix:
    the same keys and JSON files from helpers.similarity_auroc (AUROC on a score grid, with its error bound) and the nearest
    article from top_k_similar(k=1)."""
    from dae_rnn_news_recommendation_b200 import helpers
    out = {}
    print('calculate similarity')
    in_metric = 'cosine' if F.input_format == 'binary' else 'linear kernel'   # tf-idf rows are already l2-normalised (:314)
    in_name = 'binary_count' if F.input_format == 'binary' else 'tfidf'
    suffix = '(Category)' if F.label == 'category_publish_name' else '(Story)'
    all_rows = getattr(F, 'eval_all_rows', False)
    for split, X, E, lab in (('', trX, enc, trL), ('_validate', vlX, enc_v, vlL)):
        if X is None or X.shape[0] < 2 or (X.shape[0] > max_rows and not all_rows):
            print('similarity%s skipped: %s rows' % (split, None if X is None else X.shape[0]))
            continue
        large = X.shape[0] > max_rows
        for name, data, metric in ((in_name, X, in_metric), ('encoded', E, 'cosine')):
            key = 'similarity_boxplot_%s%s%s' % (name, split, suffix)
            if large:
                out[key] = helpers.similarity_auroc(data, lab, metric=metric, title=key, save_path=model.plot_dir + key + '.png')
                print('%s: AUROC %.4f (±%.1e)  related median %.4f  unrelated median %.4f' % (
                    key, out[key]['auroc'], out[key]['auroc_error_bound'], out[key]['related'].get('median', float('nan')),
                    out[key]['unrelated'].get('median', float('nan'))))
                continue
            sim = helpers.pairwise_similarity(data, metric=metric, to_host=False)
            out[key] = helpers.visualize_pairwise_similarity(lab, sim, plot='boxplot', title=key, save_path=model.plot_dir + key + '.png')
            print('%s: AUROC %.4f  related median %.4f  unrelated median %.4f' % (
                key, out[key]['auroc'], out[key]['related'].get('median', float('nan')), out[key]['unrelated'].get('median', float('nan'))))
            del sim
        if large:   # nearest_neighbors' 8192 x N block would be 32 GB at 10^6 rows
            idx, score = (a[:, 0] for a in helpers.top_k_similar(E, k=1, metric='cosine'))
        else:
            idx, score = helpers.nearest_neighbors(E, metric='cosine')
        out['nearest' + split] = (idx, score)
        for i in range(min(3, len(idx))):
            print('article %d%s: most similar %d (cosine %.4f)' % (i, split, idx[i], score[i]))
    print('calculate similarity done')
    return out


def recommend_top_k(F, model, enc, enc_v, trL, vlL):
    """--top_k K: the K most similar training articles of every training article (itself left out) and of every validation
    article (recommendations for new articles), by cosine similarity of the embeddings, at any number of rows.  Both lists
    are saved under data_dir as article_top_k_{index,score}[_validate].npy; the label precision of each is returned."""
    from dae_rnn_news_recommendation_b200 import helpers
    out = {}
    print('calculate top %d similar articles' % F.top_k)
    for split, E, lab in (('', enc, trL), ('_validate', enc_v, vlL)):
        if E is None or E.shape[0] == 0:
            continue
        idx, score = helpers.top_k_similar(E, k=F.top_k, corpus=None if split == '' else enc, metric='cosine', long_lists=F.long_lists)
        np.save(model.data_dir + 'article_top_k_index' + split, idx)
        np.save(model.data_dir + 'article_top_k_score' + split, score)
        out['top_k' + split] = (idx, score)
        out['top_k_precision' + split] = helpers.label_precision_at_k(idx, lab, trL)
        print('top %d%s: label precision %.4f' % (F.top_k, split, out['top_k_precision' + split]))
        for i in range(min(3, len(idx))):
            print('article %d%s: most similar %s' % (i, split, ', '.join('%d (%.4f)' % (j, s) for j, s in zip(idx[i], score[i]) if j >= 0)))
    return out


def recommend_top_k_input(F, model, trX, vlX, trL, vlL, emb_out):
    """--top_k_input: the same K-best lists ranked by the input vectors instead of the embeddings -- the bag-of-words baseline the
    embedding is meant to beat -- with the metric evaluate() uses for them (cosine for binary, linear kernel for tf-idf), on the
    sparse top-k kernel.  Saved as article_top_k_input_{index,score}[_validate].npy; both precisions are printed side by side."""
    from dae_rnn_news_recommendation_b200 import helpers
    out = {}
    in_metric = 'cosine' if F.input_format == 'binary' else 'linear kernel'
    print('calculate top %d similar articles by input vectors (%s)' % (F.top_k, in_metric))
    for split, X, lab in (('', trX, trL), ('_validate', vlX, vlL)):
        if X is None or X.shape[0] == 0:
            continue
        idx, score = helpers.top_k_similar(X, k=F.top_k, corpus=None if split == '' else trX, metric=in_metric)
        np.save(model.data_dir + 'article_top_k_input_index' + split, idx)
        np.save(model.data_dir + 'article_top_k_input_score' + split, score)
        out['top_k_input' + split] = (idx, score)
        out['top_k_input_precision' + split] = helpers.label_precision_at_k(idx, lab, trL)
        print('top %d%s label precision: embedding %.4f  input vectors %.4f' % (
            F.top_k, split, emb_out.get('top_k_precision' + split, float('nan')), out['top_k_input_precision' + split]))
    return out


def recommend_top_k_dedup(F, model, enc, enc_v, trL, vlL, histories, targets, emb_out):
    """--top_k_dedup T: the --top_k lists with at most one article per story.  The training articles are grouped by
    helpers.similar_pairs(enc, T) + duplicate_groups; top_k_similar / recommend then take each group's best article only (and
    recommend leaves out every group a user has read).  Saved as article_top_k_dedup_{index,score}[_validate].npy and
    user_top_k_dedup_{index,score}.npy; the label precision (hit rate / recall with --user_targets) is printed next to the plain
    lists' (emb_out)."""
    from dae_rnn_news_recommendation_b200 import helpers
    out = {}
    i, j, _ = helpers.similar_pairs(enc, F.top_k_dedup, metric='cosine')
    groups = helpers.duplicate_groups(i, j, enc.shape[0])
    n_groups = int(np.unique(groups).size)
    print('calculate top %d similar articles, one per duplicate group (cosine >= %g: %d groups of %d articles)'
          % (F.top_k, F.top_k_dedup, n_groups, enc.shape[0]))
    for split, E, lab in (('', enc, trL), ('_validate', enc_v, vlL)):
        if E is None or E.shape[0] == 0:
            continue
        idx, score = helpers.top_k_similar(E, k=F.top_k, corpus=None if split == '' else enc, metric='cosine', groups=groups,
                                           long_lists=F.long_lists)
        np.save(model.data_dir + 'article_top_k_dedup_index' + split, idx)
        np.save(model.data_dir + 'article_top_k_dedup_score' + split, score)
        out['top_k_dedup' + split] = (idx, score)
        out['top_k_dedup_precision' + split] = helpers.label_precision_at_k(idx, lab, trL)
        print('top %d%s label precision: one per group %.4f  plain %.4f' % (
            F.top_k, split, out['top_k_dedup_precision' + split], emb_out.get('top_k_precision' + split, float('nan'))))
    if histories is not None:
        idx, score = helpers.recommend(histories, enc, k=F.top_k, groups=groups, long_lists=F.long_lists)
        np.save(model.data_dir + 'user_top_k_dedup_index', idx)
        np.save(model.data_dir + 'user_top_k_dedup_score', score)
        if targets is not None:
            r = helpers.recommendation_recall(idx, targets)
            out.update({'user_dedup_hit_rate': r['hit_rate'], 'user_dedup_recall': r['recall']})
            print('users, one per group: hit rate@%d %.4f recall@%d %.4f  plain: hit rate %.4f recall %.4f (%d users with targets)' % (
                F.top_k, r['hit_rate'], F.top_k, r['recall'], emb_out.get('user_hit_rate', float('nan')),
                emb_out.get('user_recall', float('nan')), r['users']))
    return out


def find_duplicates(F, model, X, X_v, trL, vlL, metric, name, emb_out=None):
    """--dedup_threshold T: every pair of training rows of X with similarity >= T (self) and every (validation, training) pair
    (corpus), through helpers.similar_pairs, without the similarity matrix.  Saved under data_dir as <name>[_validate].npz with
    i, j, score and group (helpers.duplicate_groups of the query rows; for the validation set the components link validation rows
    through the training rows they match, and carry the smallest validation row index); the pair count, the groups of two or more
    articles and the precision / recall against the labels are returned and printed (next to emb_out's when given)."""
    from dae_rnn_news_recommendation_b200 import helpers
    out = {}
    key = name[len('article_'):]
    print('find near-duplicate articles (%s, %s >= %g)' % (key, metric, F.dedup_threshold))
    for split, Q, lab in (('', X, trL), ('_validate', X_v, vlL)):
        if Q is None or Q.shape[0] == 0:
            continue
        i, j, score = helpers.similar_pairs(Q, F.dedup_threshold, corpus=None if split == '' else X, metric=metric)
        # validation: components of the graph on validation rows 0 .. Nv-1 and training rows Nv .. Nv+Nt-1
        off = 0 if split == '' else Q.shape[0]
        g_all = helpers.duplicate_groups(i, j + off, Q.shape[0] + (0 if split == '' else X.shape[0]))
        group = g_all[:Q.shape[0]]
        np.savez(model.data_dir + name + split + '.npz', i=i, j=j, score=score, group=group)
        agree = helpers.pair_label_agreement(i, j, lab, None if split == '' else trL)
        stats = {'pairs': int(i.shape[0]), 'groups': int((np.bincount(g_all) >= 2).sum()), 'precision': agree['precision'],
                 'recall': agree['recall']}
        out[key + split] = stats
        line = '%s%s: %d pairs, %d groups of >= 2 articles, label precision %.4f recall %.4f' % (
            key, split, stats['pairs'], stats['groups'], stats['precision'], stats['recall'])
        if emb_out is not None and ('duplicates' + split) in emb_out:
            e = emb_out['duplicates' + split]
            line += '  (embedding: %d pairs, %d groups, precision %.4f recall %.4f)' % (e['pairs'], e['groups'], e['precision'], e['recall'])
        print(line)
    return out


def load_user_files(F, n_train):
    """--user_histories / --user_targets: the save_npz matrices, checked against the training set's row count before training."""
    import scipy.sparse as sp
    out = []
    for flag, path in (('--user_histories', F.user_histories), ('--user_targets', F.user_targets)):
        if not path:
            out.append(None)
            continue
        m = sp.load_npz(path)
        if m.ndim != 2 or m.shape[1] != n_train:
            raise ValueError('%s %s: shape %s, [users x %d training articles] expected' % (flag, path, m.shape, n_train))
        out.append(m)
    if out[1] is not None and out[1].shape[0] != out[0].shape[0]:
        raise ValueError('--user_targets has %d users, --user_histories %d' % (out[1].shape[0], out[0].shape[0]))
    return out


def recommend_users(F, model, enc, histories, targets):
    """--user_histories: the --top_k best unread training articles of every user from the profile of the embeddings of the
    articles the user read (helpers.recommend), saved under data_dir as user_top_k_{index,score}.npy; with --user_targets the hit
    rate and recall of the held-out reads are returned and printed."""
    from dae_rnn_news_recommendation_b200 import helpers
    print('recommend %d unread articles to %d users' % (F.top_k, histories.shape[0]))
    idx, score = helpers.recommend(histories, enc, k=F.top_k, long_lists=F.long_lists)
    np.save(model.data_dir + 'user_top_k_index', idx)
    np.save(model.data_dir + 'user_top_k_score', score)
    out = {}
    if targets is not None:
        r = helpers.recommendation_recall(idx, targets)
        out = {'user_hit_rate': r['hit_rate'], 'user_recall': r['recall']}
        print('users: hit rate@%d %.4f recall@%d %.4f (%d users with targets)' % (F.top_k, r['hit_rate'], F.top_k, r['recall'], r['users']))
    return out


def recommend_users_input(F, model, trX, histories, targets, emb_out):
    """--user_top_k_input with --user_histories: the --top_k best unread training articles of every user from the bag-of-words
    profile of the articles read (helpers.recommend_sparse, with --top_k_input's metric), saved under data_dir as
    user_top_k_input_{index,score}.npy; with --user_targets the hit rate and recall are returned and printed next to the
    embedding profile's (emb_out)."""
    from dae_rnn_news_recommendation_b200 import helpers
    in_metric = 'cosine' if F.input_format == 'binary' else 'linear kernel'
    print('recommend %d unread articles to %d users from their input vectors (%s)' % (F.top_k, histories.shape[0], in_metric))
    idx, score = helpers.recommend_sparse(histories, trX, k=F.top_k, metric=in_metric)
    np.save(model.data_dir + 'user_top_k_input_index', idx)
    np.save(model.data_dir + 'user_top_k_input_score', score)
    out = {}
    if targets is not None:
        r = helpers.recommendation_recall(idx, targets)
        out = {'user_input_hit_rate': r['hit_rate'], 'user_input_recall': r['recall']}
        print('users: hit rate@%d embedding %.4f input vectors %.4f; recall@%d embedding %.4f input vectors %.4f (%d users with '
              'targets)' % (F.top_k, emb_out.get('user_hit_rate', float('nan')), r['hit_rate'], F.top_k,
                            emb_out.get('user_recall', float('nan')), r['recall'], r['users']))
    return out


def recommend_users_sequences_input(F, trX, seqs, impressions, emb_out):
    """--user_top_k_input with --user_sequences: the bag-of-words baseline of the sequence users.  With targets, the hit rate and
    recall of helpers.recommend_sparse over each user's reads (user_input_seq_*); with --user_test_impressions, the impression
    metrics of the bag-of-words profiles of the reads before each impression (helpers.impression_metrics_sparse, user_input_imp_*).
    Printed next to the user encoder's and the mean profile's (emb_out)."""
    import scipy.sparse as sp
    from dae_rnn_news_recommendation_b200 import helpers
    from dae_rnn_news_recommendation_b200.user_model import history_matrix, prefix_histories
    indptr, items, targets = seqs
    in_metric = 'cosine' if F.input_format == 'binary' else 'linear kernel'
    cell = F.user_cell
    out = {}
    if targets is not None:
        n_u, n = len(indptr) - 1, trX.shape[0]
        has = targets >= 0
        tg = sp.csr_matrix((np.ones(int(has.sum()), np.float32), (np.flatnonzero(has), targets[has])), shape=(n_u, n))
        idx, _ = helpers.recommend_sparse(history_matrix(indptr, items, n), trX, k=F.top_k, metric=in_metric)
        r = helpers.recommendation_recall(idx, tg)
        out.update({'user_input_seq_hit_rate': r['hit_rate'], 'user_input_seq_recall': r['recall']})
        print('users: hit rate@%d %s %.4f mean profile %.4f input vectors %.4f; recall@%d %s %.4f mean profile %.4f input vectors '
              '%.4f (%d users with targets)' % (
                  F.top_k, cell.upper(), emb_out.get('user_%s_hit_rate' % cell, float('nan')),
                  emb_out.get('user_mean_hit_rate', float('nan')), r['hit_rate'], F.top_k, cell.upper(),
                  emb_out.get('user_%s_recall' % cell, float('nan')), emb_out.get('user_mean_recall', float('nan')), r['recall'],
                  r['users']))
    test_imp = impressions[1]
    if test_imp is not None:
        prof = helpers.sparse_profiles(prefix_histories((indptr, items), test_imp, trX.shape[0]), trX, to_host=False)
        m = helpers.impression_metrics_sparse(prof, trX, test_imp, metric=in_metric)
        out.update({'user_input_imp_%s' % k.replace('@', ''): m[k] for k in ('auc', 'mrr', 'ndcg@5', 'ndcg@10')})
        nan = float('nan')
        print('test impressions: ' + '; '.join(
            '%s %s %.4f mean profile %.4f input vectors %.4f' % (
                name, cell.upper(), emb_out.get('user_%s_imp_%s' % (cell, key), nan), emb_out.get('user_mean_imp_%s' % key, nan),
                out['user_input_imp_' + key]) for key, name in (('auc', 'AUC'), ('mrr', 'MRR'), ('ndcg5', 'nDCG@5'), ('ndcg10', 'nDCG@10'))))
    return out


def load_user_sequences(F, n_train):
    """--user_sequences: (indptr, items, targets or None), checked against the training set's row count before training."""
    from dae_rnn_news_recommendation_b200.user_model import check_sequences
    z = np.load(F.user_sequences)
    indptr, items = check_sequences((z['indptr'], z['items']), n_train, '--user_sequences %s' % F.user_sequences)
    targets = None
    if 'targets' in z.files:
        targets = np.asarray(z['targets']).astype(np.int64)
        if targets.shape != (len(indptr) - 1,) or targets.max(initial=-1) >= n_train or targets.min(initial=-1) < -1:
            raise ValueError('--user_sequences %s: targets must be [users] rows of the training set or -1' % F.user_sequences)
    return indptr, items, targets


def load_user_impressions(F, n_train, seqs):
    """--user_impressions / --user_test_impressions: (train, test) impression sets (None where the flag is not given), checked
    against the training set's row count and the sequences before training."""
    from dae_rnn_news_recommendation_b200.user_model import check_impressions
    out = []
    for flag, path in (('--user_impressions', F.user_impressions), ('--user_test_impressions', F.user_test_impressions)):
        out.append(check_impressions(np.load(path), n_train, '%s %s' % (flag, path), seqs[0]) if path else None)
    return tuple(out)


def recommend_users_sequences(F, model, enc, seqs, impressions=(None, None), X=None):
    """--user_sequences: train a user encoder (--user_cell: UserGRU, UserLSTM or UserAttention) on the training embeddings, save it as
    user_<cell>.npz and the --top_k best unread articles per user as user_<cell>_top_k_{index,score}.npy; with targets, the hit
    rate and recall of the encoder's and of the mean profile's recommendations for the same reads are returned and printed.
    impressions: (train, test) from load_user_impressions; the encoder trains on train's impressions when given, and test's are
    scored by the encoder's states and by the mean profiles of the same reads.  With --user_fine_tune_articles the DAE encoder over
    the training articles X is trained with the user encoder (user_model.ArticleEncoder), saved as user_<cell>_article_encoder.npz
    with its vectors as article_encoded_fine_tuned.npy, and the user encoder's recommendations and impression scores use them."""
    import scipy.sparse as sp
    from dae_rnn_news_recommendation_b200 import helpers
    from dae_rnn_news_recommendation_b200.user_model import (ArticleEncoder, UserAttention, UserGRU, UserLSTM, history_matrix,
                                                             prefix_histories)
    indptr, items, targets = seqs
    train_imp, test_imp = impressions
    cell = F.user_cell
    label = cell.upper()
    print('train a %s user encoder on %d users (%d reads, %d epochs%s)' % (label, len(indptr) - 1, items.size, F.user_epochs,
                                                                         ', impressions' if train_imp is not None else ''))
    kw = dict(heads=F.user_heads, attention_dim=F.user_attention_dim) if cell == 'attention' else {}
    if F.user_long_term:
        kw.update(long_term_users=len(indptr) - 1, long_term_mask=F.user_long_term_mask, long_term_learning_rate=F.user_long_term_lr)
    enc_cls = {'gru': UserGRU, 'lstm': UserLSTM, 'attention': UserAttention}[cell]
    rnn = enc_cls(enc.shape[1], num_epochs=F.user_epochs, seed=max(F.seed, 0), impression_loss=F.user_impression_loss,
                  impression_negatives=F.user_negatives, deterministic=F.user_deterministic, **kw)
    art = enc
    if F.user_fine_tune_articles:
        art = ArticleEncoder(X, model.get_model_parameters(), enc_act_func=model.enc_act_func, in_scale=1.0 - F.corr_frac,
                             learning_rate=F.user_article_lr)
    rnn.fit((indptr, items), art, impressions=train_imp)
    if F.user_fine_tune_articles:
        art.save(model.data_dir + 'user_%s_article_encoder.npz' % cell)
        art = art.vectors()
        np.save(model.data_dir + 'article_encoded_fine_tuned', art)
    if train_imp is not None:
        print('impressions: %(used)d used, %(skipped)d skipped' % rnn.impression_counts)
        if F.user_impression_loss == 'softmax':
            print('impression loss: softmax over each click and %s of its non-clicks (%d clicks)' % (
                'all' if F.user_negatives == 0 else 'at most %d' % F.user_negatives, rnn.impression_counts['clicks']))
    rnn.save(model.data_dir + 'user_%s.npz' % cell)
    idx, score = rnn.recommend((indptr, items), art, k=F.top_k, long_lists=F.long_lists)
    np.save(model.data_dir + 'user_%s_top_k_index' % cell, idx)
    np.save(model.data_dir + 'user_%s_top_k_score' % cell, score)
    out = {'user_%s_train_loss' % cell: rnn.train_loss[-1] if rnn.train_loss else float('nan')}
    if targets is not None:
        n_u, n = len(indptr) - 1, enc.shape[0]
        has = targets >= 0
        tg = sp.csr_matrix((np.ones(int(has.sum()), np.float32), (np.flatnonzero(has), targets[has])), shape=(n_u, n))
        hist = history_matrix(indptr, items, n)
        r = helpers.recommendation_recall(idx, tg)
        m = helpers.recommendation_recall(helpers.recommend(hist, enc, k=F.top_k, long_lists=F.long_lists)[0], tg)
        out.update({'user_%s_hit_rate' % cell: r['hit_rate'], 'user_%s_recall' % cell: r['recall'], 'user_mean_hit_rate': m['hit_rate'],
                    'user_mean_recall': m['recall']})
        print('users (%s): hit rate@%d %.4f recall@%d %.4f; mean profile: hit rate@%d %.4f recall@%d %.4f (%d users with targets)'
              % (label, F.top_k, r['hit_rate'], F.top_k, r['recall'], F.top_k, m['hit_rate'], F.top_k, m['recall'], r['users']))
    if test_imp is not None:
        g = helpers.impression_metrics(rnn.impression_states((indptr, items), art, test_imp), art, test_imp, metric='linear kernel')
        prof = helpers.user_profiles(prefix_histories((indptr, items), test_imp, enc.shape[0]), enc)
        m = helpers.impression_metrics(prof, enc, test_imp, metric='cosine')
        for name, r in ((cell, g), ('mean', m)):
            out.update({'user_%s_imp_%s' % (name, k.replace('@', '')): r[k] for k in ('auc', 'mrr', 'ndcg@5', 'ndcg@10')})
        print('test impressions (%s): AUC %.4f MRR %.4f nDCG@5 %.4f nDCG@10 %.4f; mean profile: AUC %.4f MRR %.4f nDCG@5 %.4f '
              'nDCG@10 %.4f (%d scored, %d skipped)' % (label, g['auc'], g['mrr'], g['ndcg@5'], g['ndcg@10'], m['auc'], m['mrr'],
                                                        m['ndcg@5'], m['ndcg@10'], g['impressions'], g['skipped']))
    return out


def main(argv=None):
    F = check_flags(apply_env_overrides(build_parser().parse_args(argv)))
    print(__file__ + ': Start')
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoder, utils
    model = DenoisingAutoencoder(
        seed=F.seed, model_name=F.model_name, compress_factor=F.compress_factor, enc_act_func=F.enc_act_func,
        dec_act_func=F.dec_act_func, xavier_init=F.xavier_init, corr_type=F.corr_type, corr_frac=F.corr_frac,
        loss_func=F.loss_func, main_dir=F.main_dir, opt=F.opt, learning_rate=F.learning_rate, momentum=F.momentum,
        verbose=F.verbose, verbose_step=F.verbose_step, num_epochs=F.num_epochs, batch_size=F.batch_size, alpha=F.alpha,
        triplet_strategy=F.triplet_strategy, rng_mode=F.rng_mode, mining_block_rows=F.mining_block_rows or None,
        deterministic=True if F.deterministic else None)
    data = None
    if F.synthetic:
        trX, vlX, trL, vlL = prepare_synthetic(F)
    else:
        data = restore_uci(model) if F.restore_previous_data else prepare_uci(F, model)
        (trX, vlX), (trL, vlL) = data[F.input_format], data['label_' + F.label]
        trX, vlX, trL, vlL = trX.astype(np.float32), vlX.astype(np.float32), np.asarray(trL), np.asarray(vlL)
    histories, targets = load_user_files(F, trX.shape[0]) if F.user_histories else (None, None)
    seqs = load_user_sequences(F, trX.shape[0]) if F.user_sequences else None
    imps = load_user_impressions(F, trX.shape[0], seqs) if F.user_sequences else (None, None)
    print('fit')
    model.fit(train_set=trX, validation_set=vlX if F.validation else None, train_set_label=trL,
              validation_set_label=vlL if F.validation else None, restore_previous_model=F.restore_previous_model)
    with open(model.parameter_file, 'a+') as fh:
        for k in ('train_row', 'validate_row', 'input_format', 'label', 'restore_previous_data', 'restore_previous_model'):
            print('{}={}'.format(k, getattr(F, k)), file=fh)
    print('fit done')
    # inputs are decayed by (1 - corr_frac) at inference (reference main_autoencoder.py:289-290)
    enc = model.transform(utils.decay_noise(trX, F.corr_frac), name='article_encoded', save=F.encode_full)
    enc_v = model.transform(utils.decay_noise(vlX, F.corr_frac), name='article_encoded_validate', save=F.encode_full)
    print('encoded: train %s validate %s (train_time of the last epoch: %.3f s)' % (enc.shape, enc_v.shape, model.train_time or 0.0))
    if F.save_tsv:
        save_tsv(model, data, enc, enc_v)
    model.evaluation = evaluate(F, model, trX, vlX, trL, vlL, enc, enc_v)
    if F.top_k > 0:
        model.evaluation.update(recommend_top_k(F, model, enc, enc_v, trL, vlL))
        if F.top_k_input:
            model.evaluation.update(recommend_top_k_input(F, model, trX, vlX, trL, vlL, model.evaluation))
        if histories is not None:
            model.evaluation.update(recommend_users(F, model, enc, histories, targets))
            if F.user_top_k_input:
                model.evaluation.update(recommend_users_input(F, model, trX, histories, targets, model.evaluation))
        if seqs is not None:
            model.evaluation.update(recommend_users_sequences(F, model, enc, seqs, imps, X=trX))
            if F.user_top_k_input:
                model.evaluation.update(recommend_users_sequences_input(F, trX, seqs, imps, model.evaluation))
        if F.top_k_dedup > 0:
            model.evaluation.update(recommend_top_k_dedup(F, model, enc, enc_v, trL, vlL, histories, targets, model.evaluation))
    if F.dedup_threshold > 0:
        model.evaluation.update(find_duplicates(F, model, enc, enc_v, trL, vlL, 'cosine', 'article_duplicates'))
        if F.dedup_input:
            in_metric = 'cosine' if F.input_format == 'binary' else 'linear kernel'
            model.evaluation.update(find_duplicates(F, model, trX, vlX, trL, vlL, in_metric, 'article_duplicates_input', model.evaluation))
    print(__file__ + ': End')
    return model


if __name__ == '__main__':
    main()
