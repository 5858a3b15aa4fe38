#!/usr/bin/env python
"""CLI of the explicit-triplet estimator with the reference's flag surface (reference main_autoencoder_triplet.py:20-74) driving
the H100 DenoisingAutoencoderTriplet.

    python main_autoencoder_triplet.py --model_name uci_triplet --verbose [--data_path datasets/uci_news.snappy.parquet]
    python main_autoencoder_triplet.py --model_name syn_triplet --synthetic 20000 --num_epochs 2 --batch_size 800 --verbose

Same flag names, defaults and asserts as the reference (it has no --triplet_strategy: the triplets are explicit).  The reference
reads a private parquet path (main_autoencoder_triplet.py:120) and cannot run as shipped; here --data_path defaults to the UCI
corpus of main_autoencoder.py.  Every article gets a positive (the next article with the same label) and a negative (a random article
with another label), as datasets/articles.py:83-128 does; the (org, pos, neg) matrices share one vocabulary; the data_dir cache uses
the reference's file names (`*_pos.npz`, `*_neg.npz`, main_autoencoder_triplet.py:176-205).
"""
import numpy as np

import main_autoencoder as base


def build_parser():
    ap = base.build_parser()
    for action in list(ap._actions):     # the explicit-triplet CLI has no mining strategy flag
        if action.dest == 'triplet_strategy':
            ap._remove_action(action)
            for opt in action.option_strings:
                ap._option_string_actions.pop(opt, None)
    ap.description = __doc__
    return ap


def check_flags(F):
    F.triplet_strategy = 'none'
    return base.check_flags(F)


def pair_articles(labels, min_cate=2, rng=None):
    """For every row: index of its positive (the next row carrying the same label; the last row of a label has none) and of a
    negative (a random row of another label) -- the pairing of datasets/articles.py:83-128 on row positions.  Returns
    (pos, neg, valid); rows of labels with fewer than `min_cate` members, or without a partner, are not valid."""
    rng = np.random.RandomState() if rng is None else rng
    labels = np.asarray(labels)
    n = labels.shape[0]
    pos = np.full(n, -1, dtype=np.int64)
    neg = np.full(n, -1, dtype=np.int64)
    values, counts = np.unique(labels, return_counts=True)
    for v in values[counts >= min_cate]:
        members = np.flatnonzero(labels == v)
        others = np.flatnonzero(labels != v)
        if len(others) == 0:
            continue
        pos[members[:-1]] = members[1:]
        neg[members[:-1]] = rng.choice(others, size=len(members) - 1, replace=len(others) < len(members) - 1)
    return pos, neg, (pos >= 0) & (neg >= 0)


_SUFFIX = ('', '_pos', '_neg')


def prepare_uci_triplets(F, model=None, rng=None):
    """main_autoencoder_triplet.py:120-205 on the corpus at --data_path."""
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
    df['label_category_publish_name'] = pd.factorize(df.category_publish_name.apply(lambda s: s.lstrip('即時')))[0]
    pos, neg, valid = pair_articles(df['label_' + F.label].values, min_cate=2, rng=rng)
    keep = np.flatnonzero(valid)
    n_tr, n_va = F.train_row, F.validate_row
    tr, va = keep[:n_tr], keep[n_tr:n_tr + n_va]
    text = df.main_content.values

    def df_bound(v):
        return float(v) if v <= 1 else int(v)
    cv = CountVectorizer(min_df=df_bound(F.min_df), max_df=df_bound(F.max_df), max_features=F.max_features, binary=False)
    cv.fit(np.concatenate([text[tr], text[pos[tr]], text[neg[tr]]]))      # one vocabulary over the three roles (articles.py:131-158)
    tf = TfidfTransformer()
    counts = {'train': [cv.transform(text[i]) for i in (tr, pos[tr], neg[tr])], 'validate': [cv.transform(text[i]) for i in (va, pos[va], neg[va])]}
    tf.fit(counts['train'][0])
    d = {'articles': df.iloc[tr], 'articles_validate': df.iloc[va], 'count_vectorizer': cv, 'tfidf_transformer': tf, 'binary': {}, 'tfidf': {}}
    for split in ('train', 'validate'):
        d['tfidf'][split] = dict(zip(('org', 'pos', 'neg'), (tf.transform(m).astype(np.float32) for m in counts[split])))
        binary = []
        for m in counts[split]:
            b = m.copy().astype(np.float32)
            b.data[:] = 1.0
            binary.append(b)
        d['binary'][split] = dict(zip(('org', 'pos', 'neg'), binary))
    for lab in base._LABELS:
        d['label_' + lab] = (df['label_' + lab].iloc[tr], df['label_' + lab].iloc[va])
    if model is not None:
        dd = model.data_dir
        save_file(d['articles'], dd + 'article.snappy.parquet')
        save_file(d['articles_validate'], dd + 'article_validate.snappy.parquet')
        for lab in base._LABELS:
            save_file(d['label_' + lab][0], dd + 'article_label_%s.pkl' % lab)
            save_file(d['label_' + lab][1], dd + 'article_label_%s_validate.pkl' % lab)
        save_file(counts['train'][0], dd + 'article_count_vectorized.npz')
        save_file(counts['validate'][0], dd + 'article_count_vectorized_validate.npz')
        for name, stem in (('binary', 'article_binary_count_vectorized'), ('tfidf', 'article_tfidf_vectorized')):
            for split, mid in (('train', ''), ('validate', '_validate')):
                for role, suf in zip(('org', 'pos', 'neg'), _SUFFIX):
                    save_file(d[name][split][role], dd + stem + mid + suf + '.npz')
        joblib.dump(cv, dd + 'count_vectorizer.joblib')
        joblib.dump(tf, dd + 'tfidf_transformer.joblib')
    return d


def restore_uci_triplets(model):
    """--restore_previous_data (main_autoencoder_triplet.py:96-117)."""
    import joblib
    from dae_rnn_news_recommendation_b200.io_formats import read_file
    dd = model.data_dir
    d = {'articles': read_file(dd + 'article.snappy.parquet'), 'articles_validate': read_file(dd + 'article_validate.snappy.parquet'),
         'count_vectorizer': joblib.load(dd + 'count_vectorizer.joblib'), 'tfidf_transformer': joblib.load(dd + 'tfidf_transformer.joblib'),
         'binary': {}, 'tfidf': {}}
    for name, stem in (('binary', 'article_binary_count_vectorized'), ('tfidf', 'article_tfidf_vectorized')):
        for split, mid in (('train', ''), ('validate', '_validate')):
            d[name][split] = {role: read_file(dd + stem + mid + suf + '.npz') for role, suf in zip(('org', 'pos', 'neg'), _SUFFIX)}
    for lab in base._LABELS:
        d['label_' + lab] = (read_file(dd + 'article_label_%s.pkl' % lab, data_type='pandas_series'),
                             read_file(dd + 'article_label_%s_validate.pkl' % lab, data_type='pandas_series'))
    return d


def prepare_synthetic_triplets(F):
    """Synthetic (org, pos, neg): pos = the anchor with 30 % of its words resampled, neg = an independent article (SURVEY 8d, C5)."""
    from dae_rnn_news_recommendation_b200.synth import make_sparse
    import scipy.sparse as sp
    n, seed = F.synthetic, max(F.seed, 0)
    kind = 'binary' if F.input_format == 'binary' else 'tfidf'
    org = make_sparse(n, F.max_features, 100, kind, seed=seed)
    other = make_sparse(n, F.max_features, 100, kind, seed=seed + 1)
    neg = make_sparse(n, F.max_features, 100, kind, seed=seed + 2)
    rng = np.random.RandomState(seed)
    keep = org.copy()
    keep.data = keep.data * (rng.rand(keep.nnz) >= 0.3)
    keep.eliminate_zeros()
    fill = other.copy()
    fill.data = fill.data * (rng.rand(fill.nnz) < 0.3)
    fill.eliminate_zeros()
    pos = sp.csr_matrix(keep.maximum(fill), dtype=np.float32)
    nv = min(F.validate_row, n // 5)
    cut = n - nv
    return ({'org': org[:cut], 'pos': pos[:cut], 'neg': neg[:cut]}, {'org': org[cut:], 'pos': pos[cut:], 'neg': neg[cut:]})


def main(argv=None):
    F = check_flags(base.apply_env_overrides(build_parser().parse_args(argv)))
    print(__file__ + ': Start')
    from dae_rnn_news_recommendation_b200.autoencoder import DenoisingAutoencoderTriplet, utils
    model = DenoisingAutoencoderTriplet(
        seed=F.seed, model_name=F.model_name, compress_factor=F.compress_factor, enc_act_func=F.enc_act_func,
        dec_act_func=F.dec_act_func, xavier_init=F.xavier_init, corr_type=F.corr_type, corr_frac=F.corr_frac,
        loss_func=F.loss_func, main_dir=F.main_dir, opt=F.opt, learning_rate=F.learning_rate, momentum=F.momentum,
        verbose=F.verbose, verbose_step=F.verbose_step, num_epochs=F.num_epochs, batch_size=F.batch_size, alpha=F.alpha,
        rng_mode=F.rng_mode, deterministic=True if F.deterministic else None)
    data = None
    if F.synthetic:
        trX, vlX = prepare_synthetic_triplets(F)
    else:
        data = restore_uci_triplets(model) if F.restore_previous_data else prepare_uci_triplets(F, model)
        trX, vlX = data[F.input_format]['train'], data[F.input_format]['validate']
    print('fit')
    model.fit(train_set=trX, validation_set=vlX if F.validation else None, restore_previous_model=F.restore_previous_model)
    with open(model.parameter_file, 'a+') as fh:
        for k in ('train_row', 'validate_row', 'input_format', 'label'):
            print('{}={}'.format(k, getattr(F, k)), file=fh)
    print('fit done')
    enc = model.transform(utils.decay_noise(trX['org'], F.corr_frac), name='article_encoded', save=F.encode_full)
    enc_v = model.transform(utils.decay_noise(vlX['org'], F.corr_frac), name='article_encoded_validate', save=F.encode_full)
    print('encoded: train %s validate %s (train_time of the last epoch: %.3f s)' % (enc.shape, enc_v.shape, model.train_time or 0.0))
    if F.save_tsv:
        flat = None if data is None else {'tfidf': (data['tfidf']['train']['org'], data['tfidf']['validate']['org']),
                                          'binary': (data['binary']['train']['org'], data['binary']['validate']['org']),
                                          'articles': data['articles'], 'articles_validate': data['articles_validate']}
        base.save_tsv(model, flat, enc, enc_v)
    print(__file__ + ': End')
    return model


if __name__ == '__main__':
    main()
