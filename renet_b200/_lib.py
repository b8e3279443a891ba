"""ctypes binding of librenet_b200.so (the C-ABI declared in include/renet_b200.h).

There is NO fallback: if the shared library is missing or a call fails, a RuntimeError is raised.
PyTorch is used only for device memory and streams; raw device pointers cross the boundary.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'librenet_b200.so')

_vp, _i32, _i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64

# name -> (restype, argtypes); mirrors include/renet_b200.h one to one
SIGNATURES = {
    'renet_version': (ctypes.c_int, []),
    'renet_last_error': (ctypes.c_char_p, []),
    'renet_launch_count': (_i64, []),
    'renet_pdl_launch_count': (_i64, []),
    'renet_set_gemm_engine': (ctypes.c_int, [ctypes.c_int]),
    'renet_get_gemm_engine': (ctypes.c_int, []),
    'renet_set_deterministic': (ctypes.c_int, [ctypes.c_int]),
    'renet_get_deterministic': (ctypes.c_int, []),
    'renet_set_weight_generation': (ctypes.c_int, [_i64]),
    'renet_csr_workspace_bytes': (_i64, [_i64, _i64]),
    'renet_build_csr': (ctypes.c_int, [_vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    'renet_rgcn_block_fwd': (ctypes.c_int, [_vp] * 9 + [_i64, _i64, _i32, _i32, _i32, _i32, _i32, _vp]),
    'renet_selfloop_gemm': (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _vp]),
    'renet_selfloop_gemm_bwd': (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _vp]),
    'renet_rgcn_gather': (ctypes.c_int, [_vp] * 8 + [_i64, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    'renet_debug_stream_timing': (ctypes.c_int, [_vp]),
    'renet_debug_gemm_timing': (ctypes.c_int, [_vp]),
    'renet_debug_gemm': (ctypes.c_int, [_i32, _i32, _vp, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _i64, _i32, _i32,
                                        _i64, _i64, _i64, _vp, _i64, _vp]),
    'renet_rgcn_gather_hot': (ctypes.c_int, [_vp] * 8 + [_i64, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _i32, _vp]),
    'renet_rgcn_block_bwd': (ctypes.c_int, [_vp] * 17 + [_i64, _i64, _i32, _i32, _i32, _i32, _i32, _vp]),
    'renet_rgcn_bipartite_bwd': (ctypes.c_int, [_vp] * 14 + [_i64, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _vp]),
    'renet_readout_subgraph_workspace_bytes': (_i64, [_i64, _i64]),
    'renet_readout_subgraph': (ctypes.c_int, [_vp, _i64, _i64] + [_vp] * 12 + [_i64, _vp]),
    'renet_scatter_add_rows': (ctypes.c_int, [_vp, _vp, _vp, _i64, _i32, _vp]),
    'renet_gru_workspace_bytes': (_i64, [_i64, _i64, _i64, _i32]),
    'renet_gru_fwd': (ctypes.c_int, [_vp] * 11 + [_i32] + [_vp] * 10 + [_i64, _i64, _i64, _i32, _vp, _i64, _vp]),
    'renet_gru_bwd_workspace_bytes': (_i64, [_i64, _i64, _i64, _i32]),
    'renet_gru_bwd': (ctypes.c_int, [_vp] * 11 + [_i32] + [_vp] * 18 + [_i64, _i64, _i64, _i64, _i32, _vp, _vp, _i64, _vp]),
    'renet_gru_dropout_workspace_bytes': (_i64, [_i64, _i64, _i64, _i32]),
    'renet_gru_fwd_dropout': (ctypes.c_int, [_vp] * 12 + [_i32] + [_vp] * 10 + [_i64, _i64, _i64, _i32, ctypes.c_float, ctypes.c_uint64, _vp, _i64, _vp]),
    'renet_gru_bwd_dropout_workspace_bytes': (_i64, [_i64, _i64, _i64, _i32]),
    'renet_gru_workspace_bytes_len': (_i64, [_i64, _i64, _i64, _i32, _i32]),
    'renet_gru_bwd_workspace_bytes_len': (_i64, [_i64, _i64, _i64, _i32, _i32]),
    'renet_gru_dropout_workspace_bytes_len': (_i64, [_i64, _i64, _i64, _i32, _i32]),
    'renet_gru_bwd_dropout_workspace_bytes_len': (_i64, [_i64, _i64, _i64, _i32, _i32]),
    'renet_gru_bwd_dropout': (ctypes.c_int, [_vp] * 12 + [_i32] + [_vp] * 18 + [_i64, _i64, _i64, _i64, _i32, ctypes.c_float, ctypes.c_uint64, _vp, _vp, _i64, _vp]),
    'renet_dropout_mask': (ctypes.c_int, [ctypes.c_uint64, ctypes.c_uint64, _i64, ctypes.c_float, _vp, _vp]),
    'renet_gru_dense_fwd': (ctypes.c_int, [_vp, _i32, _vp, _i32, _vp, _vp, _vp, _i32] + [_vp] * 10 + [_i64, _i64, _i32, _vp, _i64, _vp]),
    'renet_gru_dense_bwd': (ctypes.c_int, [_vp, _i32, _vp, _i32, _vp, _vp, _vp, _i32] + [_vp] * 16 + [_i64, _i64, _i32, _vp, _vp, _i64, _vp]),
    'renet_segment_pool_fwd': (ctypes.c_int, [_vp, _vp, _i64, _i32, _i32, _vp, _vp, _vp]),
    'renet_segment_pool_bwd': (ctypes.c_int, [_vp, _vp, _vp, _i64, _i64, _i32, _i32, _vp, _vp]),
    'renet_set_host_threads': (ctypes.c_int, [ctypes.c_int]),
    'renet_host_assemble_batch': (ctypes.c_int, [_i64] + [_vp] * 14 + [_i64, _i32, _vp, _vp, _i64, _vp, _i32, _vp]),
    'renet_host_plan_batch': (ctypes.c_int, [_i64] + [_vp] * 10 + [_i64, _i32, _vp, _vp, _i64, _vp, _i32, _vp]),
    'renet_host_plan_batch_grouped': (ctypes.c_int, [_i64] + [_vp] * 11 + [_i64, _i32, _vp, _vp, _i64, _vp, _i32, _vp]),
    'renet_induce_workspace_bytes': (_i64, [_i64]),
    'renet_induce_edges': (ctypes.c_int, [_vp] * 9 + [_i64, _i64, _i64] + [_vp] * 7 + [_i64, _vp]),
    'renet_encode_fwd': (ctypes.c_int, [_vp] * 12 + [_i64, _i64, _i32] + [_vp] * 9 + [_i32] + [_vp] * 10 +
                         [_i64, _i64, _i64, _i32, _i32] + [_vp] * 6 + [_vp, _i32] + [_vp, _i64, _vp]),
    'renet_loader_create': (_vp, [_i32]),
    'renet_loader_destroy': (None, [_vp]),
    'renet_loader_submit_plan': (_i64, [_vp, _i64] + [_vp] * 10 + [_i64, _i32, _vp, _vp, _i64, _vp, _i32, _vp]),
    'renet_loader_submit_assemble': (_i64, [_vp, _i64] + [_vp] * 14 + [_i64, _i32, _vp, _vp, _i64, _vp, _i32, _vp]),
    'renet_loader_wait': (ctypes.c_int, [_vp, _i64]),
    'renet_prepare_sequences': (ctypes.c_int, [_vp, _i32, _i32, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    'renet_pack_inputs': (ctypes.c_int, [_vp] * 12 + [_i64, _i32, _vp]),
    'renet_decoder_ce_workspace_bytes': (_i64, [_i64, _i32, _i32]),
    'renet_decoder_ce_fwd': (ctypes.c_int, [_vp] * 6 + [_i64, _i32, _i32, _vp, _i64, _vp]),
    'renet_decoder_ce_bwd_workspace_bytes': (_i64, [_i64, _i32, _i32]),
    'renet_decoder_ce_bwd': (ctypes.c_int, [_vp] * 5 + [ctypes.c_float] + [_vp] * 4 + [_i64, _i32, _i32, _vp, _i64, _vp]),
    'renet_decoder_soft_ce_workspace_bytes': (_i64, [_i64, _i32, _i32]),
    'renet_decoder_soft_ce_fwd': (ctypes.c_int, [_vp] * 4 + [_i64] + [_vp] * 3 + [_i64, _i32, _i32, _vp, _i64, _vp]),
    'renet_decoder_soft_ce_bwd_workspace_bytes': (_i64, [_i64, _i32, _i32]),
    'renet_decoder_soft_ce_bwd': (ctypes.c_int, [_vp] * 4 + [_i64] + [_vp] * 2 + [ctypes.c_float] + [_vp] * 4 +
                                  [_i64, _i32, _i32, _vp, _i64, _vp]),
    'renet_decoder_group_topk_workspace_bytes': (_i64, [_i64, _i32, _i32, _i32, _i32]),
    'renet_decoder_group_topk': (ctypes.c_int, [_vp] * 4 + [_i64, _i32, _i32, _i32, _i32, _i32, _i32] + [_vp] * 4 +
                                 [_i64, _vp]),
    'renet_decoder_topk_workspace_bytes': (_i64, [_i64, _i32, _i32, _i32]),
    'renet_decoder_topk': (ctypes.c_int, [_vp] * 6 + [_i64, _i32, _i32, _i32, _i32] + [_vp] * 4 + [_i64, _vp]),
    'renet_decoder_rank_workspace_bytes': (_i64, [_i64, _i32, _i32]),
    'renet_decoder_rank': (ctypes.c_int, [_vp] * 9 + [_i64, _i32, _i32, _vp, _i64, _vp]),
    'renet_decoder_rank_multi': (ctypes.c_int, [_vp] * 4 + [_i32] + [_vp] * 5 + [_i64, _i32, _i32, _vp, _i64, _vp]),
    'renet_grad_sumsq_workspace_bytes': (_i64, []),
    'renet_grad_sumsq': (ctypes.c_int, [_vp, _i64, _vp, _i32, _vp, _i64, _vp]),
    'renet_adam_step': (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64] + [ctypes.c_float] * 5 + [_i64, _vp, ctypes.c_float, ctypes.c_float, _vp]),
}

_lib = None


def lib():
    """The loaded library; raises if it has not been built (python -m renet_b200.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                'renet_b200: %s is missing -- build it with `python -m renet_b200.build` '
                '(there is no CPU or PyTorch fallback for the hot path)' % LIB_PATH)
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)     # AttributeError if the .so does not export the symbol
            fn.restype, fn.argtypes = res, args
        _lib = handle
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().renet_last_error().decode('utf-8', 'replace')
        raise RuntimeError('renet_b200: %s failed (status %d): %s' % (what, rc, msg))


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())


def stream():
    """The current CUDA stream of the current device as a raw handle.  (torch.cuda.current_stream() costs ~10 us of Python per
    call -- device-index checks, a Stream object -- and the e2e path asks 18 times per step; the raw getter is ~0.3 us.)

    Every kernel call asks for its stream here, so this is also where the library's deterministic mode follows
    torch.use_deterministic_algorithms(): the flag is read on every call and passed on when it has changed."""
    dev = torch._C._cuda_getDevice()
    det = torch.are_deterministic_algorithms_enabled()
    if det != _deterministic[0]:
        lib().renet_set_deterministic(int(det))
        _deterministic[0] = det
    return ctypes.c_void_p(torch._C._cuda_getCurrentRawStream(dev))


_deterministic = [False]       # the value last passed to renet_set_deterministic (the library starts at 0)


def pinned_slots(pool, words):
    """Refill a deque of pinned int32[words] read-back slots in bulk: one cudaHostAlloc for 1024 slots instead of one per
    batch inside a timed loop (a slot returns to its pool when its value has been read)."""
    block = torch.empty(1024 * words, dtype=torch.int32).pin_memory()
    pool.extend(block[i * words:(i + 1) * words] for i in range(1024))


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError('renet_b200: the hot path runs on CUDA only (got a %s tensor); '
                               'there is no CPU fallback' % t.device)


def launch_count():
    return int(lib().renet_launch_count())


def pdl_launch_count():
    return int(lib().renet_pdl_launch_count())


# ---- packed-weight cache (renet_set_weight_generation) -----------------------------------------------------------------
_pack_tokens = __import__('itertools').count(1)


def new_pack_token():
    """Unique id of a module instance: part of its weight generation, so that another module whose parameters happen to
    be allocated at the same addresses can never hit this one's packed images."""
    return next(_pack_tokens)


_weight_epoch = [0]


def invalidate_packed_weights():
    """Declare that weights may have changed in a way the in-place version counters do not see (updates through
    ``p.data``, raw-pointer optimiser kernels, load_state_dict into re-pointed storage ...): every packed image made so
    far becomes stale.  Pure host bookkeeping -- the epoch is part of every weight generation."""
    _weight_epoch[0] += 1


class weight_generation:
    """Context manager: while active, the tensor-core GEMM engine may reuse packed weight images made under the same
    generation = hash(module token, invalidation epoch, (address, in-place version) of every weight).  Outside of it the
    cache is off, so direct C-ABI callers are never served a stale image.  Only version-bumping in-place updates are
    tracked automatically; anything else must call ``invalidate_packed_weights()`` (the trainer in parallel.py does)."""

    def __init__(self, token, params):
        self.gen = hash((token, _weight_epoch[0]) + tuple((p.data_ptr(), p._version) for p in params)) & ((1 << 62) - 1)

    def __enter__(self):
        lib().renet_set_weight_generation(self.gen)

    def __exit__(self, *exc):
        lib().renet_set_weight_generation(-1)
        return False
