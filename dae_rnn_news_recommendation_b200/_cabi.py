"""ctypes binding of libdae_sm100.so (the C-ABI library declared in include/dae_sm100.h).

There is no CPU fallback: if the library is missing or a call fails, this raises.
"""
import ctypes
import ctypes as C
import os
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ.get('DAE_SM100_LIB', _PKG / 'libdae_sm100.so'))

ACT = {'none': 0, 'sigmoid': 1, 'tanh': 2}
LOSS = {'cross_entropy': 0, 'mean_squared': 1, 'cosine_proximity': 2}
STRATEGY = {'none': 0, 'batch_all': 1, 'batch_hard': 2, 'explicit': 3}
OPT = {'gradient_descent': 0, 'ada_grad': 1, 'momentum': 2, 'adam': 3}
STAT = {'cost': 0, 'ae_loss': 1, 'triplet_loss': 2, 'fraction': 3, 'num': 4, 'sum_w': 5, 'n_valid': 6, 'sum_lw': 7,
        'triplet_sum': 8, 'n_active': 9}
STAT_SLOTS = 16
MAX_TRIPLET_BATCH = 32768   # DAE_MAX_TRIPLET_BATCH: largest batch_all / batch_hard batch (S, G and G's bf16 copy: ~13 GB)
MAX_BLOCKED_BATCH = 262144  # DAE_MAX_BLOCKED_BATCH: largest batch of a block-mined engine (TrainEngine(mining_block_rows=R))


def act_code(name):
    """autoencoder/autoencoder.py:380-387: anything that is not 'sigmoid'/'tanh' is the identity."""
    return ACT.get(name, 0)


p, i32, i64, f32, u64, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_uint64, C.c_size_t

_SIGNATURES = {
    'dae_version': (C.c_int, []),
    'dae_last_error': (C.c_int, [C.c_char_p, sz]),
    'dae_batch_prepare': (C.c_int, [p, i64, p, i32, p, i32, p, p, p, p, p, p, p]),
    'dae_batch_prepare_next': (C.c_int, [p, i64, i64, p, i32, p, i32, p, p, p, p, p, p, p]),
    'dae_batch_prepare_blocked': (C.c_int, [p, i64, p, i32, p, i32, p, p, p, p, p, p, p]),
    'dae_batch_prepare_next_blocked': (C.c_int, [p, i64, i64, p, i32, p, i32, p, p, p, p, p, p, p]),
    'dae_batch_commit': (C.c_int, [i32, p, p, p, p, p, p, p, p, p, p, p, p, p]),
    'dae_batch_prepare_explicit': (C.c_int, [p, i64, p, i32, i64, p, p, p]),
    'dae_step_advance': (C.c_int, [p, i64, p]),
    'dae_encode_csr_fwd': (C.c_int, [p, p, p, p, i32, i32, i32, f32, p, p, i32, p, i64, p, p, p, i64, p]),
    'dae_encode_csr_fwd_hot': (C.c_int, [p, p, p, i32, i32, i32, f32, p, p, i32, p, i64, p, p, i32, i32, p]),
    'dae_col_scan': (C.c_int, [p, i32, p, p, p]),
    'dae_encode_csr_bwd_gather': (C.c_int, [p, p, p, p, i32, i32, i32, f32, p, p, i32, p, p, i64, p, p, i32, p, p, p, p, p, p, p]),
    'dae_encode_csr_bwd': (C.c_int, [p, p, p, p, i32, i32, i32, f32, p, p, i32, p, p, i64, p, p, i32, p]),
    'dae_sgemm': (C.c_int, [i32, i32, i32, f32, p, i64, i64, p, i64, i64, f32, p, i64, p]),
    'dae_split_bf16': (C.c_int, [p, i32, i32, i64, p, p, i64, i32, f32, p]),
    'dae_sym_split_bf16': (C.c_int, [p, i32, i64, f32, p, p, i64, p]),
    'dae_gemm_bf16x3': (C.c_int, [i32, i32, i32, f32, p, p, i64, i32, p, p, i64, i32, p, i64, i32, i32, p, i32, i32, p]),
    'dae_gemm_config': (C.c_int, [i32, i32]),
    'dae_decode_prepare': (C.c_int, [i32, i32, p, p, p, p, p, p]),
    'dae_decode_fused_bf16x3': (C.c_int, [i32, i32, i32, p, p, i64, p, p, i64, p, p, p, p, p, i32, i32, p, p, p, p, i64, p, p, i32, p]),
    'dae_reduce_parts': (C.c_int, [p, i32, i32, p, p]),
    'dae_decode_loss_bwd': (C.c_int, [p, p, p, p, i32, i32, p, i32, i32, p, p, p, i64, p, p]),
    'dae_colsum': (C.c_int, [p, i32, i32, i64, p, p]),
    'dae_triplet_batch_all': (C.c_int, [p, i64, i32, p, p, p, i64, p, i32, p, p, i64, p]),
    'dae_triplet_config': (C.c_int, [i32]),
    'dae_gemm_sym_bf16x3': (C.c_int, [i32, i32, f32, p, p, i64, p, p, i64, p, i64, i32, p]),
    'dae_triplet_batch_hard': (C.c_int, [p, i64, i32, p, p, i64, p, p, p]),
    'dae_triplet_batch_all_rows': (C.c_int, [p, i64, i32, i32, i32, p, p, p, i64, p, i32, p, p, i64, p]),
    'dae_triplet_batch_hard_rows': (C.c_int, [p, i64, i32, i32, i32, p, p, i64, p, p, p]),
    'dae_triplet_batch_hard_finish': (C.c_int, [p, i32, p, p, i32, i64, p]),
    'dae_triplet_explicit': (C.c_int, [p, p, p, i32, i32, i64, f32, p, p, p, p, p]),
    'dae_step_finalize': (C.c_int, [p, p, i32, p, i32, i32, f32, p, p, p, p]),
    'dae_optimizer_step': (C.c_int, [p, p, p, p, i64, i32, f32, f32, f32, i32, p, p, p, i32, i32, i64, p]),
    'dae_rownorm_split_bf16': (C.c_int, [p, i32, i32, i64, i32, p, p, i64, p, i64, p]),
    'dae_row_argmax': (C.c_int, [p, i32, i32, i64, i64, i32, p, p, p]),
    'dae_similarity_topk_bf16x3': (C.c_int, [i32, i32, i32, p, p, i64, p, p, i64, i32, i64, i32, i32, p, i64, p, p, p]),
    'dae_similarity_topk_workspace': (C.c_int, [i32, i32, i32, i32, p]),
    'dae_csr_similarity_topk': (C.c_int, [p, p, p, i32, i64, i32, p, p, p, i32, i64, i32, i32, i64, i32, i32, p, i64, p, p, p]),
    'dae_csr_similarity_topk_workspace': (C.c_int, [i32, i32, i64, i32, i32, i32, p]),
    'dae_similarity_topk_excl_bf16x3': (C.c_int, [i32, i32, i32, p, p, i64, p, p, i64, i32, i64, i32, i32, p, i64, p, p, p, p, i64, p]),
    'dae_csr_similarity_topk_excl': (C.c_int, [p, p, p, i32, i64, i32, p, p, p, i32, i64, i32, i32, i64, i32, i32, p, i64, p, p, p, p,
                                               i64, p]),
    'dae_similarity_topk_groups_bf16x3': (C.c_int, [i32, i32, i32, p, p, i64, p, p, i64, i32, i64, i32, i32, p, i64, p, p, p, p, i64, p,
                                                    p]),
    'dae_csr_similarity_topk_groups': (C.c_int, [p, p, p, i32, i64, i32, p, p, p, i32, i64, i32, i32, i64, i32, i32, p, i64, p, p, p, p,
                                                 i64, p, p]),
    'dae_similarity_topk_bound_bf16x3': (C.c_int, [i32, i32, i32, p, p, i64, p, p, i64, i32, i64, i32, i32, p, i64, p, p, i64, p, p,
                                                   p]),
    'dae_similarity_topk_bound_workspace': (C.c_int, [i32, i32, i32, i32, p]),
    'dae_similarity_topk_collect_bf16x3': (C.c_int, [i32, i32, i32, p, p, i64, p, p, i64, i64, i32, p, p, p, i64, p, p, i64, p, p, p,
                                                     p]),
    'dae_similarity_topk_select': (C.c_int, [i32, i64, p, p, p, i32, p, p, p, p]),
    'dae_pair_partition': (C.c_int, [p, i64, i32, p, p, p, p, p]),
    'dae_auroc_count': (C.c_int, [p, i64, p, i64, i32, p, p]),
    'dae_similarity_pair_hist_bf16x3': (C.c_int, [i32, i32, p, p, i64, p, f32, i32, p, p, p]),
    'dae_csr_similarity_pair_hist': (C.c_int, [p, p, p, i32, i64, i32, p, f32, i32, p, i64, p, p, p]),
    'dae_csr_similarity_pair_hist_workspace': (C.c_int, [i32, i64, i32, p]),
    'dae_similarity_pairs_bf16x3': (C.c_int, [i32, i32, i32, p, p, i64, p, p, i64, i32, f32, p, i64, p, p, p, p]),
    'dae_csr_similarity_pairs': (C.c_int, [p, p, p, i32, i64, i32, p, p, p, i32, i64, i32, i32, f32, p, i64, p, i64, p, p, p, p]),
    'dae_csr_similarity_pairs_workspace': (C.c_int, [i32, i32, i64, i32, p]),
    'dae_pairs_sort': (C.c_int, [i64, i32, i32, p, p, p, p, p, i64, p, p]),
    'dae_pairs_sort_workspace': (C.c_int, [i64, i32, p]),
    'dae_allreduce_multimem': (C.c_int, [p, p, p, i32, i32, i64, i32, p]),
    'dae_mask_values': (C.c_int, [p, p, i64, f32, u64, u64, p, p]),
    'dae_salt_pepper_csr': (C.c_int, [p, p, p, i64, i64, i32, i64, f32, f32, p, u64, u64, p, p, p, i64, p, p, sz, p]),
    'dae_salt_pepper_workspace': (C.c_int, [i64, p]),
    # GRU user encoder
    'dae_gather_split_bf16': (C.c_int, [p, i64, p, i32, i32, p, p, i64, i32, p]),
    'dae_gru_cell_fwd': (C.c_int, [i32, i32, p, i64, p, i64, p, i64, p, i64, i32, p, p, i64, p, i64, p]),
    'dae_gru_cell_bwd': (C.c_int, [i32, i32, p, i64, p, i64, p, i64, p, i64, p, p, p, p, i64, p]),
    'dae_seq_negatives': (C.c_int, [p, i64, i32, u64, u64, u64, p, p]),
    'dae_seq_rank_loss': (C.c_int, [p, i64, p, i64, i32, p, p, i64, f32, p, i64, p, p]),
    # LSTM user encoder
    'dae_lstm_cell_fwd': (C.c_int, [i32, i32, p, i64, p, i64, p, i64, p, i64, p, i64, i32, p, p, i64, p, i64, p]),
    'dae_lstm_cell_bwd': (C.c_int, [i32, i32, p, i64, p, i64, p, i64, p, i64, p, i64, p, i64, p, p, i64, p]),
    # long-term user vectors
    'dae_rows_optimizer_step': (C.c_int, [p, i64, i32, p, i32, p, i64, p, p, p, i32, f32, f32, p]),
    # attention user encoder
    'dae_seq_attention_fwd': (C.c_int, [i32, i32, p, p, i32, i32, p, i64, p, i64, p, p, i64, p, i64, p]),
    'dae_seq_attention_bwd': (C.c_int, [i32, i32, p, p, i32, i32, p, i64, p, i64, p, i64, p, i64, p, p, i64, p]),
    'dae_seq_pool_fwd': (C.c_int, [i32, i32, p, p, i32, i32, p, i64, p, p, i64, p, i64, p, p, p]),
    'dae_seq_pool_bwd': (C.c_int, [i32, i32, p, p, i32, i32, p, i64, p, i64, p, i64, p, i64, p, p, p, p, i64, p, p, i64, p, p, p]),
    # impression logs
    'dae_impression_rank_loss': (C.c_int, [p, i64, p, i64, i32, p, i64, p, p, p, f32, p, i64, p, p]),
    'dae_impression_metrics': (C.c_int, [p, i64, p, i64, i32, i32, p, p, p, i64, p, p, p]),
    'dae_impression_softmax_loss': (C.c_int, [p, i64, p, i64, i32, p, i64, p, p, p, p, i32, u64, u64, f32, p, i64, p, p, p]),
    # article encoder fine-tuned through the user encoders' losses
    'dae_encode_csr_fwd_groups': (C.c_int, [p, p, p, p, i32, i32, i32, f32, p, p, i32, p, i64, p, p, p, i64, i32, p]),
    'dae_seq_rank_loss_grad': (C.c_int, [p, i64, p, i64, i32, p, p, i64, f32, p, i64, p, p, i64, p]),
    'dae_impression_rank_loss_grad': (C.c_int, [p, i64, p, i64, i32, p, i64, p, p, p, f32, p, i64, p, p, i64, p]),
    'dae_impression_softmax_loss_grad': (C.c_int, [p, i64, p, i64, i32, p, i64, p, p, p, p, i32, u64, u64, f32, p, i64, p, p, p, i64,
                                                   p]),
    'dae_touch_compact_workspace': (C.c_int, [i64, p]),
    'dae_touch_compact': (C.c_int, [p, i64, C.c_uint32, p, p, p, p, p, p]),
    'dae_rows_scatter_add': (C.c_int, [p, i64, p, i64, i32, p, i64, p]),
    # bag-of-words user profiles
    'dae_csr_profiles_count': (C.c_int, [p, p, i32, i32, p, p, i32, p, p]),
    'dae_csr_profiles': (C.c_int, [p, p, p, i32, i32, p, p, p, i32, p, i32, i32, i32, p, p, p]),
    'dae_csr_impression_metrics': (C.c_int, [p, p, p, p, p, p, i32, i32, i32, p, p, p, i64, p, p, p]),
    # deterministic training step
    'dae_gemm_det_workspace': (C.c_int, [p]),
    'dae_gemm_bf16x3_det': (C.c_int, [i32, i32, i32, f32, p, p, i64, i32, p, p, i64, i32, p, i64, i32, i32, p, i32, i32, p, i64, p]),
    'dae_gemm_sym_bf16x3_det': (C.c_int, [i32, i32, f32, p, p, i64, p, p, i64, p, i64, i32, p, i64, p]),
    'dae_decode_loss_parts': (C.c_int, [i32, p]),
    'dae_decode_fused_bf16x3_det': (C.c_int, [i32, i32, i32, p, p, i64, p, p, i64, p, p, p, p, p, i32, i32, p, p, p, p, i64, p, p, i32,
                                              p]),
    'dae_encode_csr_bwd_det_workspace': (C.c_int, [i32, i32, i32, i64, p]),
    'dae_encode_csr_bwd_det': (C.c_int, [p, p, p, p, i32, i32, i32, f32, p, p, i32, p, p, i64, p, p, i64, p, i64, p]),
    'dae_encode_sparse_dw_add': (C.c_int, [i32, i32, i32, i64, p, i64, p, p]),
    'dae_triplet_batch_all_det': (C.c_int, [p, i64, i32, p, p, p, i64, p, i32, p, p, i64, p, p]),
    'dae_triplet_batch_hard_det': (C.c_int, [p, i64, i32, p, p, i64, p, p, p, p]),
    'dae_triplet_batch_all_rows_det': (C.c_int, [p, i64, i32, i32, i32, p, p, p, i64, p, i32, p, p, i64, p, p]),
    'dae_triplet_batch_hard_rows_det': (C.c_int, [p, i64, i32, i32, i32, p, p, i64, p, p, p, p]),
    'dae_triplet_explicit_det': (C.c_int, [p, p, p, i32, i32, i64, f32, p, p, p, p, p, p]),
    'dae_triplet_loss_sum': (C.c_int, [p, i32, p, p]),
    # deterministic user-encoder training
    'dae_seq_rank_loss_det': (C.c_int, [p, i64, p, i64, i32, p, p, i64, f32, p, i64, p, p]),
    'dae_seq_rank_loss_grad_det': (C.c_int, [p, i64, p, i64, i32, p, p, i64, f32, p, i64, p, p, p, p, p]),
    'dae_impression_rank_loss_det': (C.c_int, [p, i64, p, i64, i32, p, i64, p, p, p, f32, p, i64, p, p]),
    'dae_impression_rank_loss_grad_det': (C.c_int, [p, i64, p, i64, i32, p, i64, p, p, p, f32, p, i64, p, p, p, p, p]),
    'dae_impression_softmax_loss_det': (C.c_int, [p, i64, p, i64, i32, p, i64, p, p, p, p, i32, u64, u64, f32, p, i64, p, p, p]),
    'dae_impression_softmax_loss_grad_det': (C.c_int, [p, i64, p, i64, i32, p, i64, p, p, p, p, i32, u64, u64, f32, p, i64, p, p, p, p,
                                                       p, p]),
    'dae_loss_slots_sum': (C.c_int, [p, i64, p, p]),
    'dae_ordered_rows_workspace': (C.c_int, [i64, i64, i32, p]),
    'dae_ordered_rows': (C.c_int, [p, p, p, i64, p, i64, p, i64, p, i64, i32, i32, p, i64, p, i64, p]),
}


def query(name, *args, ctype=C.c_int64):
    """Call a size query export whose last argument is an output scalar; returns that scalar."""
    out = ctype(0)
    call(name, *args, ctypes.addressof(out))
    return int(out.value)

_lib = None


class DaeError(RuntimeError):
    pass


def exported_symbols():
    """Every symbol include/dae_sm100.h declares (used by the CPU-side export test)."""
    return list(_SIGNATURES)


def lib():
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise DaeError('%s not found: build it with `python -m dae_rnn_news_recommendation_b200.build` '
                           '(there is no CPU fallback)' % LIB_PATH)
        l = ctypes.CDLL(str(LIB_PATH))
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def last_error():
    buf = ctypes.create_string_buffer(512)
    lib().dae_last_error(buf, 512)
    return buf.value.decode()


def call(name, *args):
    rc = getattr(lib(), name)(*args)
    if rc != 0:
        raise DaeError('%s failed (%d): %s' % (name, rc, last_error()))


def ptr(t):
    """device pointer of a torch tensor (None -> NULL)"""
    return None if t is None else t.data_ptr()
