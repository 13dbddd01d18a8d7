"""ctypes binding of the C ABI declared in include/cotr_b200.h.

There is deliberately no CPU fallback: if the shared library is missing or no sm_90 GPU is visible the calls raise.
"""
import ctypes
import os

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libcotr_b200.so")

_lib = None


class CotrTensor(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char_p), ("data", ctypes.POINTER(ctypes.c_float)),
                ("ndim", ctypes.c_int32), ("shape", ctypes.c_int64 * 4)]


class TestGemmDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in (
        "path", "M", "N", "K", "a_mode", "lda", "H", "W", "C", "OH", "OW", "KH", "KW", "stride", "pad",
        "relu", "add_period", "ld_add", "ldr", "ldc", "a_ln", "res_ln", "emit_part", "reserved")] + [("a_elems", ctypes.c_int64)] + \
        [(n, ctypes.c_int32) for n in ("out_rows", "res_rows", "res_col0", "n_pairs", "n_images", "redirect", "n_vt", "vt_pairs")] + \
        [("blk_map", ctypes.c_int32 * 12)] + \
        [(n, ctypes.c_int32) for n in ("force_bn", "force_ksplit", "plan_bn", "plan_loader", "plan_dln", "plan_ksplit",
                                        "plan_grid_x", "plan_grid_y", "plan_ln_defused", "reserved2")]


class TestAttentionDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in (
        "path", "nq", "npairs", "operands", "slots", "slot", "ctx_pairs", "pair0", "q_rows", "ldq", "q_col0", "n_tiles",
        "key_split", "maps_rows", "maps_row0", "reserved")]


class TestMlpDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("M", "rows", "split", "in_place")]


class RefineGroup(ctypes.Structure):
    _fields_ = [("image_from", ctypes.c_int32), ("image_to", ctypes.c_int32), ("first", ctypes.c_int32), ("count", ctypes.c_int32),
                ("s_from", ctypes.c_double), ("s_to", ctypes.c_double)]


class LaunchRecord(ctypes.Structure):
    _fields_ = [("kernel", ctypes.c_int32), ("M", ctypes.c_int32), ("N", ctypes.c_int32), ("K", ctypes.c_int32),
                ("ms", ctypes.c_float)]


KERNEL_NAMES = ("gemm_tc", "gemm_simt", "attention_tc", "attention_simt", "layernorm", "maxpool", "query_encode", "stem_canvas", "gemm_mlp",
                "attention_weights_tc", "attention_weights_simt", "match_queries", "match_pixels", "nearest", "mutual",
                "refine_geometry", "resize_h", "resize_v", "refine_step", "grouped_candidates", "group_tasks", "dense_first_guess",
                "resize_image", "resize_maps")

# name -> (restype, argtypes); every symbol include/cotr_b200.h declares
_PROTOTYPES = {
    "cotr_create": (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(CotrTensor), ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]),
    "cotr_destroy": (None, [ctypes.c_void_p]),
    "cotr_context_create": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]),
    "cotr_context_destroy": (None, [ctypes.c_void_p]),
    "cotr_encode_context": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_decode": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_encode_context_attention": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                                     ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_decode_attention": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                             ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_encode_images": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_encode_context_pairs": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                                 ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_decode_ragged": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                          ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_mutual_nearest": (ctypes.c_int, [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_match_keypoints": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                            ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                            ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_forward": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_forward_host": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "cotr_preprocess": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                       ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_refine": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                   ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_double]
                    + [ctypes.c_void_p] * 8),
    "cotr_refine_grouped": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int64,
                                           ctypes.c_double] + [ctypes.c_void_p] * 7),
    "cotr_dense_postprocess": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_flow_tile_merge": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p] + [ctypes.c_int] * 6 +
                             [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]),
    "cotr_group_tasks": (ctypes.c_int, [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_dense_first_guess": (ctypes.c_int, [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                              ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                              ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_dense_first_guess_f32": (ctypes.c_int, [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                  ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                  ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_resize_image": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                         ctypes.c_int, ctypes.c_void_p]),
    "cotr_resize_maps": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                        ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "cotr_rasterize_triangles": (ctypes.c_int, [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_exchange_create": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]),
    "cotr_exchange_handle": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_exchange_connect": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "cotr_exchange_connect_local": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p)]),
    "cotr_exchange_push": (ctypes.c_longlong, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "cotr_exchange_wait": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t), ctypes.c_void_p]),
    "cotr_exchange_status": (ctypes.c_int, [ctypes.c_void_p]),
    "cotr_exchange_destroy": (None, [ctypes.c_void_p]),
    "cotr_set_graph_mode": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    "cotr_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int]),
    "cotr_last_launch_count": (ctypes.c_int, [ctypes.c_void_p]),
    "cotr_profile_begin": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    "cotr_profile_end": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(LaunchRecord), ctypes.c_int]),
    "cotr_debug_read": (ctypes.c_int64, [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p, ctypes.c_int64]),
    "cotr_set_gemm_path": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    "cotr_test_gemm": (ctypes.c_int, [ctypes.POINTER(TestGemmDesc)] + [ctypes.c_void_p] * 12),
    "cotr_test_attention": (ctypes.c_int, [ctypes.POINTER(TestAttentionDesc)] + [ctypes.c_void_p] * 6),
    "cotr_test_mlp": (ctypes.c_int, [ctypes.POINTER(TestMlpDesc)] + [ctypes.c_void_p] * 10),
    "cotr_test_rowwise": (ctypes.c_int, [ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 6),
    "cotr_test_refine_math": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double] + [ctypes.c_void_p] * 4),
    "cotr_test_pilot_boxes": (ctypes.c_int, [ctypes.c_int, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 3),
    "cotr_debug_set_variant": (None, [ctypes.c_int]),
    "cotr_last_error": (ctypes.c_char_p, []),
    "cotr_version": (ctypes.c_char_p, []),
}


def lib():
    """The loaded shared library (loads on first use; raises if it has not been built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `python -m cotr_b200.build` "
                               "(cotr_b200 has no CPU / PyTorch fallback by design)")
        handle = ctypes.CDLL(LIB_PATH)
        for name, (restype, argtypes) in _PROTOTYPES.items():
            try:
                fn = getattr(handle, name)
            except AttributeError:
                if os.environ.get("COTR_B200_ALLOW_OLD_LIB"):       # A/B against a build of an older revision
                    continue
                raise
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = handle
    return _lib


def last_error():
    return lib().cotr_last_error().decode("utf-8", "replace")


def check(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what} failed: {last_error()}")


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


class NativeContext:
    """Decoder K/V cache of up to `max_pairs` encoded image pairs (cotr_context)."""

    def __init__(self, model, max_pairs):
        self.model = model
        self.max_pairs = max_pairs
        self.pairs = 0
        h = ctypes.c_void_p()
        check(lib().cotr_context_create(model.handle, int(max_pairs), ctypes.byref(h)), "cotr_context_create")
        self.handle = h

    def close(self):
        # cotr_context_destroy only frees the context's own K/V buffers; it never touches the (possibly already
        # destroyed) model, so it is called unconditionally - skipping it leaked 12.6 MB per pair.
        if self.handle is not None:
            lib().cotr_context_destroy(self.handle)
        self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class NativeModel:
    """Owner of a `cotr_model` handle built from a reference-schema state dict (CPU fp32 tensors / arrays)."""

    def __init__(self, state_dict, device_index):
        if not torch.cuda.is_available():
            raise RuntimeError("cotr_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        names, arrays = [], []
        for k, v in state_dict.items():
            a = v.detach().to("cpu", torch.float32).contiguous().numpy() if isinstance(v, torch.Tensor) else np.ascontiguousarray(v, np.float32)
            if a.ndim > 4:
                continue
            names.append(k.encode())
            arrays.append(a)
        arr = (CotrTensor * len(arrays))()
        for i, (n, a) in enumerate(zip(names, arrays)):
            arr[i].name = n
            arr[i].data = a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
            arr[i].ndim = a.ndim
            for d in range(a.ndim):
                arr[i].shape[d] = a.shape[d]
        h = ctypes.c_void_p()
        self.handle = None
        self.device_index = int(device_index)
        check(lib().cotr_create(self.device_index, arr, len(arrays), ctypes.byref(h)), "cotr_create")
        self.handle = h

    # ---- calls ------------------------------------------------------------------------------------
    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device_index).cuda_stream)

    def forward(self, img, queries):
        B, Q = queries.shape[0], queries.shape[1]
        pred = torch.empty((B, Q, 2), dtype=torch.float32, device=img.device)
        check(lib().cotr_forward(self.handle, _ptr(img), _ptr(queries), B, Q, _ptr(pred), self._stream()), "cotr_forward")
        return pred

    def encode_context(self, img, ctx):
        check(lib().cotr_encode_context(self.handle, _ptr(img), img.shape[0], ctx.handle, self._stream()), "cotr_encode_context")
        ctx.pairs = img.shape[0]

    def decode(self, ctx, queries):
        B, Q = queries.shape[0], queries.shape[1]
        pred = torch.empty((B, Q, 2), dtype=torch.float32, device=queries.device)
        check(lib().cotr_decode(self.handle, ctx.handle, _ptr(queries), B, Q, _ptr(pred), self._stream()), "cotr_decode")
        return pred

    def decode_ragged(self, ctx, queries, offsets):
        """Pair p's queries are rows offsets[p] .. offsets[p+1]-1 of the packed (R,2) device tensor `queries`, R = offsets[B];
        offsets: B+1 integers (host) -> packed (R,2) predictions (cotr_decode_ragged)."""
        off = np.ascontiguousarray(offsets, dtype=np.int64).reshape(-1)
        R = max(int(off[-1]), 0) if off.size else 0          # the library checks the offsets
        pred = torch.empty((R, 2), dtype=torch.float32, device=queries.device)
        check(lib().cotr_decode_ragged(self.handle, ctx.handle, _ptr(queries), ctypes.c_void_p(off.ctypes.data), off.size - 1,
                                       _ptr(pred), self._stream()), "cotr_decode_ragged")
        return pred

    def match_keypoints(self, feat, sizes, kpts, kpt_offsets, pairs, ctx):
        """Cached features (2,N,256,1024) + (N,2) int (W,H) sizes + packed (sum K_i,2) fp64 device keypoints with N+1 host
        offsets + (B,2) pairs -> (corr (R,2) fp64, nearest (R,) int32, match (R,2) int32, count (B,) int32) on the device,
        in the row layout of cotr_match_keypoints; ctx needs room for 2B pairs."""
        off, pairs, R = _match_layout(kpt_offsets, pairs)
        sizes = np.ascontiguousarray(sizes, dtype=np.int32)
        B = pairs.shape[0]
        corr = torch.empty((R, 2), dtype=torch.float64, device=kpts.device)
        nearest, match, count = _match_outputs(R, B, kpts.device)
        check(lib().cotr_match_keypoints(self.handle, _ptr(feat), feat.shape[1], ctypes.c_void_p(sizes.ctypes.data), _ptr(kpts),
                                         ctypes.c_void_p(off.ctypes.data), ctypes.c_void_p(pairs.ctypes.data), B, ctx.handle,
                                         _ptr(corr), _ptr(nearest), _ptr(match), _ptr(count), self._stream()), "cotr_match_keypoints")
        ctx.pairs = 2 * B
        return corr, nearest, match, count

    def encode_context_attention(self, img, ctx, layer_mask):
        """encode_context that also returns the head-averaged attention maps of the encoder layers selected by
        `layer_mask` (bit l = layer l): (popcount(layer_mask), B, 512, 512) fp32 (cotr_encode_context_attention)."""
        B = img.shape[0]
        attn = torch.empty((bin(layer_mask).count("1"), B, 512, 512), dtype=torch.float32, device=img.device)
        check(lib().cotr_encode_context_attention(self.handle, _ptr(img), B, ctx.handle, int(layer_mask),
                                                  _ptr(attn) if layer_mask else None, self._stream()), "cotr_encode_context_attention")
        ctx.pairs = B
        return attn

    def encode_images(self, images):
        """(N,3,256,256) fp32 device images -> their backbone features, a (2, N, 256, 1024) float16 device tensor
        (plane, image, 16x16 position, channel: COTR_IMAGE_FEATURE_BYTES per image) (cotr_encode_images)."""
        N = images.shape[0]
        feat = torch.empty((2, N, 256, 1024), dtype=torch.float16, device=images.device)
        check(lib().cotr_encode_images(self.handle, _ptr(images), N, _ptr(feat), self._stream()), "cotr_encode_images")
        return feat

    def encode_context_pairs(self, feat, pairs, ctx):
        """Encode the pairs (B,2) of images of `feat` (from encode_images) into ctx (cotr_encode_context_pairs)."""
        self.encode_context_pairs_attention(feat, pairs, ctx, 0)

    def encode_context_pairs_attention(self, feat, pairs, ctx, layer_mask):
        """encode_context_pairs that also returns the encoder attention maps selected by `layer_mask`, as
        encode_context_attention does: (popcount(layer_mask), B, 512, 512) fp32."""
        pairs = np.ascontiguousarray(pairs, dtype=np.int32)
        B = pairs.shape[0]
        attn = torch.empty((bin(layer_mask).count("1"), B, 512, 512), dtype=torch.float32, device=feat.device)
        check(lib().cotr_encode_context_pairs(self.handle, _ptr(feat), feat.shape[1], ctypes.c_void_p(pairs.ctypes.data), B,
                                              ctx.handle, int(layer_mask), _ptr(attn) if layer_mask else None, self._stream()),
              "cotr_encode_context_pairs")
        ctx.pairs = B
        return attn

    def decode_attention(self, ctx, queries, layer_mask):
        """decode that also returns the head-averaged attention maps of the decoder layers selected by `layer_mask`:
        -> (pred (B,Q,2), maps (popcount(layer_mask), B, Q, 512) fp32) (cotr_decode_attention)."""
        B, Q = queries.shape[0], queries.shape[1]
        pred = torch.empty((B, Q, 2), dtype=torch.float32, device=queries.device)
        attn = torch.empty((bin(layer_mask).count("1"), B, Q, 512), dtype=torch.float32, device=queries.device)
        check(lib().cotr_decode_attention(self.handle, ctx.handle, _ptr(queries), B, Q, int(layer_mask),
                                          _ptr(attn) if layer_mask else None, _ptr(pred), self._stream()), "cotr_decode_attention")
        return pred, attn

    def forward_host(self, img_np, queries_np, out_np=None):
        """Host buffers in, host buffer out (H2D + forward + D2H inside the C call)."""
        B, Q = queries_np.shape[0], queries_np.shape[1]
        if out_np is None:
            out_np = np.empty((B, Q, 2), dtype=np.float32)
        check(lib().cotr_forward_host(self.handle, ctypes.c_void_p(img_np.ctypes.data), ctypes.c_void_p(queries_np.ctypes.data),
                                      B, Q, ctypes.c_void_p(out_np.ctypes.data)), "cotr_forward_host")
        return out_np

    def preprocess(self, img_from_dev, img_to_dev, rects):
        """uint8 HWC device images + (n,6) int32 crop rectangles -> (n,3,256,512) fp32 normalised canvases (device)."""
        rects = np.ascontiguousarray(rects, dtype=np.int32)
        n = rects.shape[0]
        canvas = torch.empty((n, 3, 256, 512), dtype=torch.float32, device=img_from_dev.device)
        check(lib().cotr_preprocess(self.handle, _ptr(img_from_dev), img_from_dev.shape[0], img_from_dev.shape[1],
                                    _ptr(img_to_dev), img_to_dev.shape[0], img_to_dev.shape[1],
                                    ctypes.c_void_p(rects.ctypes.data), n, _ptr(canvas), self._stream()), "cotr_preprocess")
        return canvas

    def refine(self, images, groups, zooms, batch, wave, max_good, rel_threshold, loc_from, loc_to):
        """The zoom-in walk (cotr_refine).  images: uint8 HWC device tensors; groups: (image_from, image_to, first,
        count, s_from, s_to) tuples; loc_from / loc_to: (n,2) fp64 device tensors ->
        (history (n,L+1,2) fp64, rects (n,L,6) int32, good (n,) int32 on the device, walked, (code, chunk, level))."""
        n, L = loc_from.shape[0], len(zooms)
        ptrs = (ctypes.c_void_p * len(images))(*[t.data_ptr() for t in images])
        hw = np.ascontiguousarray([[t.shape[0], t.shape[1]] for t in images], dtype=np.int32)
        tab = (RefineGroup * len(groups))(*[RefineGroup(*g) for g in groups])
        z = np.ascontiguousarray(zooms, dtype=np.float64)
        history = torch.empty((n, L + 1, 2), dtype=torch.float64, device=loc_from.device)
        rects = torch.empty((n, max(L, 1), 6), dtype=torch.int32, device=loc_from.device)
        good = torch.zeros((max(n, 1),), dtype=torch.int32, device=loc_from.device)[:n]
        walked = ctypes.c_int64(0)
        status = (ctypes.c_int32 * 3)()
        check(lib().cotr_refine(self.handle, ptrs, ctypes.c_void_p(hw.ctypes.data), len(images), tab, len(groups),
                                ctypes.c_void_p(z.ctypes.data), L, int(batch), int(wave), int(max_good), float(rel_threshold),
                                _ptr(loc_from), _ptr(loc_to), _ptr(history), _ptr(rects), _ptr(good), ctypes.byref(walked),
                                status, self._stream()), "cotr_refine")
        return history, rects, good, walked.value, tuple(status)

    def refine_grouped(self, img_from, img_to, s_from, s_to, zooms, level, ids, batch_size, max_load, max_good, rel_threshold,
                       loc_from, history, rects, good):
        """One grouped batch (cotr_refine_grouped).  img_*: uint8 HWC device tensors; ids: the level's open tasks in shuffled
        order; loc_from (n,2) fp64, history (n,L+1,2) fp64, rects (n,L,6) int32, good (n+1,) int32: device tensors the
        batches of one walk share -> (squad (n_ids,) int32 numpy, (n_squads, longest, num_steps, stepped, status))."""
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        z = np.ascontiguousarray(zooms, dtype=np.float64)
        squad = np.empty(max(ids.size, 1), dtype=np.int32)
        result = (ctypes.c_int32 * 5)()
        check(lib().cotr_refine_grouped(self.handle, _ptr(img_from), img_from.shape[0], img_from.shape[1], _ptr(img_to), img_to.shape[0],
                                        img_to.shape[1], float(s_from), float(s_to), ctypes.c_void_p(z.ctypes.data), z.size, int(level),
                                        ctypes.c_void_p(ids.ctypes.data), ids.size, loc_from.shape[0], int(batch_size), int(max_load),
                                        int(max_good), float(rel_threshold), _ptr(loc_from), _ptr(history), _ptr(rects), _ptr(good),
                                        ctypes.c_void_p(squad.ctypes.data), result, self._stream()), "cotr_refine_grouped")
        return squad[:ids.size], tuple(result)

    def dense_postprocess(self, pred_dev):
        """(n, 131072, 2) fp32 predictions of the dense grid queries -> (n, 256, 512, 3) [x, y, confidence] (device)."""
        pred_dev = pred_dev.contiguous()
        n = pred_dev.shape[0]
        out = torch.empty((n, 256, 512, 3), dtype=torch.float32, device=pred_dev.device)
        check(lib().cotr_dense_postprocess(self.handle, _ptr(pred_dev), n, _ptr(out), self._stream()), "cotr_dense_postprocess")
        return out

    def flow_tile_merge(self, tile, affine, patch, flow, conf, first):
        """One 256 x 256 x 3 tile answer (a view into dense_postprocess' output) -> affine, Pillow-exact float resize to
        the patch size, confidence merge into the (oh,ow,2) / (oh,ow) device canvases (cotr_flow_tile_merge)."""
        assert tile.is_cuda and tile.dtype == torch.float32 and tile.shape == (256, 256, 3) and tile.stride(2) == 1 and tile.stride(1) == 3
        aff = np.ascontiguousarray(affine, dtype=np.float64).reshape(6)
        check(lib().cotr_flow_tile_merge(self.handle, _ptr(tile), int(tile.stride(0)), ctypes.c_void_p(aff.ctypes.data),
                                         int(patch.x), int(patch.y), int(patch.w), int(patch.h), int(patch.ow), int(patch.oh),
                                         _ptr(flow), _ptr(conf), int(bool(first)), self._stream()), "cotr_flow_tile_merge")

    def resize_image(self, img, size):
        """(H,W,3) uint8 CUDA image -> (H',W',3) uint8, Pillow's bilinear resize to size = (H',W') (cotr_resize_image)."""
        assert img.is_cuda and img.dtype == torch.uint8 and img.ndim == 3 and img.shape[2] == 3
        img = img.contiguous()
        out = torch.empty((int(size[0]), int(size[1]), 3), dtype=torch.uint8, device=img.device)
        check(lib().cotr_resize_image(self.handle, _ptr(img), img.shape[0], img.shape[1], _ptr(out), out.shape[0], out.shape[1],
                                      self._stream()), "cotr_resize_image")
        return out

    def resize_maps(self, maps, size):
        """(H,W) or (H,W,C) fp32 CUDA maps, C = 1 .. 3 -> the same layout at size = (H',W'), bit for bit
        utils.float_image_resize (cotr_resize_maps)."""
        assert maps.is_cuda and maps.dtype == torch.float32 and maps.ndim in (2, 3)
        src = maps.contiguous()
        c = src.shape[2] if src.ndim == 3 else 1
        out = torch.empty((int(size[0]), int(size[1])) + tuple(src.shape[2:]), dtype=torch.float32, device=src.device)
        check(lib().cotr_resize_maps(self.handle, _ptr(src), src.shape[0], src.shape[1], c, _ptr(out), out.shape[0], out.shape[1],
                                     self._stream()), "cotr_resize_maps")
        return out

    def set_graph_mode(self, enabled):
        check(lib().cotr_set_graph_mode(self.handle, int(bool(enabled))), "cotr_set_graph_mode")

    def set_gemm_path(self, path):
        check(lib().cotr_set_gemm_path(self.handle, int(path)), "cotr_set_gemm_path")

    def last_launch_count(self):
        return lib().cotr_last_launch_count(self.handle)

    def profile_begin(self, max_records=4096):
        check(lib().cotr_profile_begin(self.handle, int(max_records)), "cotr_profile_begin")
        self._prof_max = int(max_records)

    def profile_end(self):
        """-> list of (kernel name, M, N, K, ms) for every launch since profile_begin, in launch order."""
        buf = (LaunchRecord * self._prof_max)()
        rc = lib().cotr_profile_end(self.handle, buf, self._prof_max)
        if rc > 0:
            raise RuntimeError(f"cotr_profile_end failed: {last_error()}")
        n = -rc - 1
        return [(KERNEL_NAMES[buf[i].kernel], buf[i].M, buf[i].N, buf[i].K, buf[i].ms) for i in range(n)]

    def debug_read(self, name, n_elems):
        out = np.empty(int(n_elems), dtype=np.float32)
        n = lib().cotr_debug_read(self.handle, name.encode(), ctypes.c_void_p(out.ctypes.data), int(n_elems))
        if n < 0:
            raise RuntimeError(f"cotr_debug_read({name}) failed")
        return out[:n]

    def close(self):
        if self.handle is not None:
            lib().cotr_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


EXCHANGE_HANDLE_BYTES = 64


class NativeExchange:
    """One rank's end of the peer-memory result exchange (cotr_exchange, include/cotr_b200.h): `push` writes this rank's
    block into every peer's buffer over NVLink, `wait` gathers one step's blocks in rank order.  Connecting is the
    caller's job: `handle()` -> all-gather the 64-byte handles between the processes -> `connect(handles)`; exchanges
    living in one process use `connect_local(all_exchanges)`."""

    def __init__(self, device_index, rank, world, block_bytes, slots=4):
        self.device_index, self.rank, self.world, self.block_bytes, self.slots = int(device_index), int(rank), int(world), int(block_bytes), int(slots)
        h = ctypes.c_void_p()
        check(lib().cotr_exchange_create(self.device_index, self.rank, self.world, self.block_bytes, self.slots, ctypes.byref(h)), "cotr_exchange_create")
        self.handle_ = h

    def handle(self):
        buf = ctypes.create_string_buffer(EXCHANGE_HANDLE_BYTES)
        check(lib().cotr_exchange_handle(self.handle_, buf), "cotr_exchange_handle")
        return buf.raw

    def connect(self, handles):
        """handles: the `handle()` of every rank, in rank order."""
        blob = b"".join(handles)
        assert len(blob) == self.world * EXCHANGE_HANDLE_BYTES
        check(lib().cotr_exchange_connect(self.handle_, ctypes.create_string_buffer(blob, len(blob))), "cotr_exchange_connect")

    def connect_local(self, exchanges):
        arr = (ctypes.c_void_p * self.world)(*[e.handle_ for e in exchanges])
        check(lib().cotr_exchange_connect_local(self.handle_, arr), "cotr_exchange_connect_local")

    def _stream(self, stream):
        s = stream if stream is not None else torch.cuda.current_stream(self.device_index)
        return ctypes.c_void_p(s.cuda_stream)

    def push(self, block, stream=None):
        """block: contiguous CUDA tensor of this rank (at most block_bytes, a multiple of 16 bytes).  Returns the step number."""
        assert block.is_cuda and block.is_contiguous() and block.device.index == self.device_index
        seq = lib().cotr_exchange_push(self.handle_, _ptr(block), block.numel() * block.element_size(), self._stream(stream))
        if seq < 0:
            raise RuntimeError(f"cotr_exchange_push failed: {last_error()}")
        return int(seq)

    def wait(self, seq, out=None, bytes_per_rank=None, stream=None):
        """Enqueue the wait for step `seq`; `out` (contiguous CUDA tensor, or None) receives the blocks in rank order."""
        sizes = None
        if bytes_per_rank is not None:
            sizes = (ctypes.c_size_t * self.world)(*[int(b) for b in bytes_per_rank])
        need = sum(int(b) for b in bytes_per_rank) if bytes_per_rank is not None else self.world * self.block_bytes
        if out is not None:
            assert out.is_cuda and out.is_contiguous() and out.numel() * out.element_size() >= need
        check(lib().cotr_exchange_wait(self.handle_, int(seq), _ptr(out) if out is not None else None, sizes, self._stream(stream)), "cotr_exchange_wait")

    def status(self):
        return int(lib().cotr_exchange_status(self.handle_))

    def close(self):
        if self.handle_:
            lib().cotr_exchange_destroy(self.handle_)
            self.handle_ = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def group_tasks(pts, boxes, batch_size, max_load, device):
    """(n,4) end points + (n,8) pilot boxes (float64 numpy, list order) -> (squad (n,), rank (n,), n_squads): the device
    version of FasterSparseEngine's squad formation (cotr_group_tasks)."""
    n = int(pts.shape[0])
    dev = torch.device(device)
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    p = torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float64)).to(dev)
    b = torch.from_numpy(np.ascontiguousarray(boxes, dtype=np.float64)).to(dev)
    out = torch.empty(2 * n + 1, dtype=torch.int32, device=dev)
    stream = ctypes.c_void_p(torch.cuda.current_stream(idx).cuda_stream)
    check(lib().cotr_group_tasks(idx, _ptr(p), _ptr(b), n, int(batch_size), int(max_load), _ptr(out), ctypes.c_void_p(out.data_ptr() + 4 * n),
                                 ctypes.c_void_p(out.data_ptr() + 8 * n), stream), "cotr_group_tasks")
    host = out.cpu().numpy()
    return host[:n], host[n:2 * n], int(host[2 * n])


def _match_layout(kpt_offsets, pairs):
    """-> (int64 offsets, int32 (B,2) pairs, R rows of the call); R = 0 when the table is malformed (the library reports it)."""
    off = np.ascontiguousarray(kpt_offsets, dtype=np.int64).reshape(-1)
    pairs = np.ascontiguousarray(pairs, dtype=np.int32).reshape(-1, 2)
    n = off.size - 1
    R = 0
    if n >= 1 and pairs.size and (pairs >= 0).all() and (pairs < n).all() and (np.diff(off) >= 0).all():
        R = int(np.diff(off)[pairs].sum())
    return off, pairs, R


def _match_outputs(R, B, device):
    """nearest (R,), match (R,2), count (B,): int32 device tensors"""
    return (torch.empty((R,), dtype=torch.int32, device=device), torch.empty((R, 2), dtype=torch.int32, device=device),
            torch.empty((B,), dtype=torch.int32, device=device))


def mutual_nearest(kpts, kpt_offsets, pairs, corr):
    """Packed (sum K_i,2) fp64 device keypoints with N+1 host offsets + (B,2) pairs + (R,2) fp64 device pixel predictions
    in the row layout of cotr_mutual_nearest -> (nearest (R,) int32, match (R,2) int32, count (B,) int32) on the device."""
    off, pairs, R = _match_layout(kpt_offsets, pairs)
    dev = kpts.device.index if kpts.device.index is not None else torch.cuda.current_device()
    nearest, match, count = _match_outputs(R, pairs.shape[0], kpts.device)
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    check(lib().cotr_mutual_nearest(dev, _ptr(kpts), ctypes.c_void_p(off.ctypes.data), off.size - 1, ctypes.c_void_p(pairs.ctypes.data),
                                    pairs.shape[0], _ptr(corr), _ptr(nearest), _ptr(match), _ptr(count), stream), "cotr_mutual_nearest")
    return nearest, match, count


def dense_first_guess(flow, conf_from, conf_to, kpts, loc_to, counts, f32_maps=False):
    """The forced first guesses of one direction (cotr_dense_first_guess).  flow (H_f,W_f,2) / conf_from (H_f,W_f) /
    conf_to (H_t,W_t): contiguous fp32 CUDA maps; kpts (n,2) float32 or float64 CUDA (x, y); outputs written in place:
    loc_to (n,2) fp64, counts (2,) int64 (pixels below THRESHOLD_AREA in conf_from, conf_to).  f32_maps: the arithmetic
    numpy does on float32 maps, as 'stretching' mode holds them (cotr_dense_first_guess_f32)."""
    for t in (flow, conf_from, conf_to, kpts, loc_to, counts):
        assert t.is_cuda and t.is_contiguous() and t.device == flow.device
    assert flow.dtype == conf_from.dtype == conf_to.dtype == torch.float32 and kpts.dtype in (torch.float32, torch.float64)
    assert flow.ndim == 3 and flow.shape[2] == 2 and tuple(conf_from.shape) == tuple(flow.shape[:2]) and conf_to.ndim == 2
    n = kpts.shape[0]
    assert kpts.shape == (n, 2) and loc_to.dtype == torch.float64 and loc_to.shape == (n, 2)
    assert counts.dtype == torch.int64 and counts.shape == (2,)
    dev = flow.device.index if flow.device.index is not None else torch.cuda.current_device()
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    name = "cotr_dense_first_guess_f32" if f32_maps else "cotr_dense_first_guess"
    check(getattr(lib(), name)(dev, _ptr(flow), _ptr(conf_from), flow.shape[0], flow.shape[1], _ptr(conf_to), conf_to.shape[0],
                               conf_to.shape[1], _ptr(kpts), int(kpts.dtype == torch.float32), n, _ptr(loc_to), _ptr(counts), stream), name)


def rasterize_triangles(tris, H, W):
    """(n_tri,3,4) fp32 CUDA tensor [x, y, u, v] per vertex -> (H,W,2) fp32 CUDA tensor (cotr_rasterize_triangles)."""
    tris = tris.contiguous()
    assert tris.is_cuda and tris.dtype == torch.float32 and tris.ndim == 3 and tris.shape[1:] == (3, 4)
    out = torch.empty((H, W, 2), dtype=torch.float32, device=tris.device)
    dev = tris.device.index if tris.device.index is not None else torch.cuda.current_device()
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    check(lib().cotr_rasterize_triangles(dev, _ptr(tris), tris.shape[0], int(H), int(W), _ptr(out), stream), "cotr_rasterize_triangles")
    return out


GEMM_LOADERS = ("gather", "im2col", "stem", "halo")
GEMM_REDIRECT = {None: 0, "vt": 1, "images": 2}


def test_gemm(path, A, w_host, *, bias=None, addmat=None, add_period=1, residual=None, res_col0=0, relu=False, ln=None,
              a_mode=0, conv=None, M=None, ldc=None, out=None, a_ln=False, res_ln=False, part_out=None, pairs=None,
              n_images=None, blk_map=None, n_vt=0, vt=None, img=None, bn=0, ksplit=0, plan=None):
    """Kernel-level hook: out = epilogue(A W^T), launched as the model launches it (cotr_test_gemm).

    A: CUDA fp32, contiguous; all of it reaches the kernel (row-major: (rows >= M, lda) with lda >= K, the columns past
    K must not be read; token gather: (n_images*256, lda) features with `pairs` an (M/512, 2) image table).
    residual: (rows >= M, ldr), the launch reads columns res_col0 .. res_col0+N-1.  out: (rows >= M, ldc >= N), rows and
    columns the launch does not write come back as passed (default: zeros of (M, ldc or N)).
    a_ln / res_ln: `ln` = (gamma, beta) is a DEFERRED LayerNorm of the A rows / of the residual rows (tensor-core path).
    blk_map (256-column blocks, GemmParams::blk_map) with n_vt slots: values transposed into vt (pairs, n_vt, 256, 512)
    fp32 (returned updated in place), or keys and values into the operand images `img` (a uint8 CUDA buffer of
    pairs * n_vt * 8 * 132096 bytes, left undecoded).  bn / ksplit (path 0): force the tile width / split-K, 0 = rule.
    plan: a dict that receives the plan the launch used (tile width, loader, dln, ksplit, grid, ln_defused)."""
    N, K = w_host.shape
    assert A.is_cuda and A.dtype == torch.float32 and A.is_contiguous()
    d = TestGemmDesc()
    d.path = path
    d.N, d.K = N, K
    d.a_mode = a_mode
    if a_mode == 0:
        d.M = A.shape[0] if M is None else M
        d.lda = A.shape[-1]
    else:
        d.M = M
        for k_, v_ in (conv or {}).items():
            setattr(d, k_, v_)
        d.lda = conv.get("C", 0) if a_mode != 3 else A.shape[-1]
    d.a_elems = A.numel()
    tab = None
    if a_mode == 3:
        tab = np.ascontiguousarray(np.arange(2 * (d.M // 512)) if pairs is None else pairs, dtype=np.int32).reshape(-1, 2)
        d.n_pairs = tab.shape[0]
        d.n_images = A.numel() // (256 * d.lda) if n_images is None else n_images
    d.relu = int(relu)
    d.a_ln = int(a_ln)
    d.res_ln = int(res_ln)
    d.emit_part = int(part_out is not None)
    d.add_period = add_period
    d.ld_add = addmat.stride(0) if addmat is not None else 0
    if residual is not None:
        assert residual.is_contiguous()
        d.ldr, d.res_rows, d.res_col0 = residual.shape[1], residual.shape[0], res_col0
    if out is None:
        out = torch.zeros((d.M, N if ldc is None else ldc), dtype=torch.float32, device=A.device)
    assert out.is_contiguous() and out.dtype == torch.float32
    d.out_rows, d.ldc = out.shape
    if blk_map is not None:
        d.redirect = GEMM_REDIRECT["images" if img is not None else "vt"]
        d.n_vt = n_vt
        buf = img if img is not None else vt
        d.vt_pairs = buf.shape[0] if vt is not None else buf.numel() // (n_vt * 8 * 132096)
        assert vt is None or (vt.is_contiguous() and tuple(vt.shape[1:]) == (n_vt, 256, 512))
        assert img is None or (img.dtype == torch.uint8 and img.is_contiguous() and img.numel() == d.vt_pairs * n_vt * 8 * 132096)
        for i, b in enumerate(blk_map):
            d.blk_map[i] = b
    d.force_bn, d.force_ksplit = bn, ksplit
    w_np = np.ascontiguousarray(w_host, np.float32)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    check(lib().cotr_test_gemm(ctypes.byref(d), p(A), ctypes.c_void_p(w_np.ctypes.data), p(bias), p(addmat), p(residual),
                               p(ln[0]) if ln else None, p(ln[1]) if ln else None, p(out), p(part_out),
                               ctypes.c_void_p(tab.ctypes.data) if tab is not None else None, p(vt), p(img)), "cotr_test_gemm")
    if plan is not None:
        plan.update(bn=d.plan_bn, loader=GEMM_LOADERS[d.plan_loader] if d.plan_bn else None, dln=d.plan_dln,
                    ksplit=d.plan_ksplit, grid=(d.plan_grid_x, d.plan_grid_y), ln_defused=d.plan_ln_defused)
    return out


ATTENTION_OPERANDS = {"rowmajor": 0, "images": 1}


def test_attention(path, q, k, v, nq, npairs, *, operands="rowmajor", pair0=0, slot=0, q_col0=0, tiles=None, key_split=0,
                   out=None, maps=None, maps_row0=0):
    """Kernel-level hook: softmax(q k^T) v per head, launched as the model launches it (cotr_test_attention).

    q: (rows, ldq) CUDA fp32, the launch reads columns q_col0 .. q_col0+255.  k, v: (ctx_pairs*512, slots*256) CUDA fp32,
    the keys / values of `slots` layers side by side per pair as in a context; the launch reads slot `slot` of pairs
    pair0 .. .  operands: "rowmajor" (fp32 SIMT schedule) or "images" (tensor-core schedule).  tiles: optional (n,3)
    table of (pair, first row, row count) - then nq / npairs are unused.  key_split (path 0): 0 = launch rule, 1 or 2.
    out: (rows,256) CUDA fp32, rows the launch does not own are returned unchanged (default zeros).
    maps: optional (maps_rows,512) CUDA fp32, written in place: the head-averaged attention maps of the same operands
    (path 0 with "images", path 1 with "rowmajor"), local pair p, query i at row maps_row0 + p*nq + i; the other rows
    are left unchanged."""
    d = TestAttentionDesc()
    d.path, d.nq, d.npairs = path, nq, npairs
    d.operands = ATTENTION_OPERANDS[operands]
    d.slots, d.slot = k.shape[1] // 256, slot
    d.ctx_pairs, d.pair0 = k.shape[0] // 512, pair0
    d.q_rows, d.ldq, d.q_col0 = q.shape[0], q.shape[1], q_col0
    d.key_split = key_split
    assert k.shape == v.shape and k.shape[0] % 512 == 0 and k.shape[1] % 256 == 0
    assert all(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() for t in (q, k, v))
    tab = None
    if tiles is not None:
        tab = np.ascontiguousarray(tiles, dtype=np.int32).reshape(-1, 3)
        d.n_tiles = tab.shape[0]
    if out is None:
        out = torch.zeros((q.shape[0], 256), dtype=torch.float32, device=q.device)
    assert out.is_contiguous() and out.shape == (q.shape[0], 256)
    if maps is not None:
        assert maps.is_cuda and maps.dtype == torch.float32 and maps.is_contiguous() and maps.ndim == 2 and maps.shape[1] == 512
        d.maps_rows, d.maps_row0 = maps.shape[0], maps_row0
    check(lib().cotr_test_attention(ctypes.byref(d), _ptr(q), _ptr(k), _ptr(v), _ptr(out),
                                    ctypes.c_void_p(tab.ctypes.data) if tab is not None else None,
                                    _ptr(maps) if maps is not None else None), "cotr_test_attention")
    return out


def test_mlp(x, M, w1, b1, w2, b2, g, be, g2=None, be2=None, *, split=0, in_place=False, out=None):
    """Kernel-level hook: the fused feed-forward block (cotr_test_mlp) on rows < M of x (rows, 256):
    LN(x + relu(x w1^T + b1) w2^T + b2), then LN(., g2, be2) when given.  w1 (1024,256) / w2 (256,1024) host arrays, the
    other operands CUDA fp32.  split: 0 = launch rule, 4 or 8 CTAs per row tile.  in_place: the launch writes into x.
    out: (rows,256), rows >= M are returned unchanged (in place: x's rows) (default zeros)."""
    d = TestMlpDesc()
    d.M, d.rows, d.split, d.in_place = M, x.shape[0], split, int(in_place)
    if out is None:
        out = torch.zeros_like(x)
    assert x.is_contiguous() and out.is_contiguous() and x.shape == out.shape and x.shape[1] == 256
    w1 = np.ascontiguousarray(w1, np.float32)
    w2 = np.ascontiguousarray(w2, np.float32)
    assert w1.shape == (1024, 256) and w2.shape == (256, 1024)
    p = lambda t: _ptr(t) if t is not None else None
    check(lib().cotr_test_mlp(ctypes.byref(d), _ptr(x), ctypes.c_void_p(w1.ctypes.data), _ptr(b1), ctypes.c_void_p(w2.ctypes.data),
                              _ptr(b2), _ptr(g), _ptr(be), p(g2), p(be2), _ptr(out)), "cotr_test_mlp")
    return out


ROWWISE_OPS = {"layernorm": 0, "layernorm_f32": 1, "layernorm_twice": 2, "query_encode": 3}


def test_rowwise(op, x, g1=None, b1=None, g2=None, b2=None):
    """Kernel-level hook: a row kernel (cotr_test_rowwise) on x (rows,256), or on (rows,2) points for query_encode
    -> (rows,256)."""
    out = torch.zeros((x.shape[0], 256), dtype=torch.float32, device=x.device)
    p = lambda t: _ptr(t) if t is not None else None
    check(lib().cotr_test_rowwise(ROWWISE_OPS[op], x.shape[0], _ptr(x), p(g1), p(b1), p(g2), p(b2), _ptr(out)), "cotr_test_rowwise")
    return out


def test_refine_math(op, inputs, ints, levels=1, rel_threshold=0.0):
    """cotr_test_refine_math: the per-task arithmetic of cotr_refine on the host (see include/cotr_b200.h).
    op 0 -> (n,4) int32 [left, top, size, flag]; 1 / 2 -> (n,2) float64; 3 -> (n,) int32 good."""
    a = np.ascontiguousarray(inputs, dtype=np.float64)
    b = np.ascontiguousarray(ints, dtype=np.int32)
    n = b.shape[0]
    out = np.zeros((n, 2), dtype=np.float64)
    out_i = np.zeros((n, 4 if op == 0 else 1), dtype=np.int32)
    check(lib().cotr_test_refine_math(int(op), n, int(levels), float(rel_threshold), ctypes.c_void_p(a.ctypes.data),
                                      ctypes.c_void_p(b.ctypes.data), ctypes.c_void_p(out.ctypes.data),
                                      ctypes.c_void_p(out_i.ctypes.data)), "cotr_test_refine_math")
    return out if op in (1, 2) else (out_i if op == 0 else out_i[:, 0])


def test_pilot_boxes(pts, geom, device=0):
    """cotr_test_pilot_boxes: the candidate kernel of cotr_refine_grouped on (n,4) fp64 end points and [h_from, w_from,
    h_to, w_to, size_from, size_to] -> ((n,8) fp64 pilot boxes, (n,) int32 crop failure codes)."""
    p = np.ascontiguousarray(pts, dtype=np.float64).reshape(-1, 4)
    g = np.ascontiguousarray(geom, dtype=np.int32)
    box = np.zeros((p.shape[0], 8), dtype=np.float64)
    fail = np.zeros(p.shape[0], dtype=np.int32)
    check(lib().cotr_test_pilot_boxes(int(device), ctypes.c_void_p(p.ctypes.data), p.shape[0], ctypes.c_void_p(g.ctypes.data),
                                      ctypes.c_void_p(box.ctypes.data), ctypes.c_void_p(fail.ctypes.data)), "cotr_test_pilot_boxes")
    return box, fail
