"""Host scheduler of the recursive zoom-in (reference: COTR/inference/sparse_engine.py).

`SparseEngine` runs one query per network context (sparse_engine.py:17-264); `FasterSparseEngine` lets nearby
tasks share the context of a "pilot" task (:267-427).  Task state, RNG call order (`np.random.choice` with
replacement in gen_tasks, `np.random.permutation` per grouped batch), truncation rules and the acceptance /
border / cycle-consistency filters follow the reference so that, driven by the same model, both produce the same
correspondences - including the reference's quirk that the faster engine strands tasks which were never grouped at
an earlier zoom level (SURVEY.md section 3.3).
"""
import math

import numpy as np
import PIL.Image
import torch

from . import refinement_task
from . import inference_helper
from .inference_helper import (THRESHOLD_SPARSE, THRESHOLD_AREA, cotr_corr_base, cotr_flow_maps, flow_on_device, get_patch_centered_at,
                               stretched_flow_maps)
from .refinement_task import RefinementTask
from ..utils import utils
from ..utils.utils import ImagePatch


def stretch_to_square_np(img):
    """Resize to max(h,w) x max(h,w) with Pillow bilinear (reference: COTR/cameras/capture.py:123-125)."""
    size = max(*img.shape[:2])
    return np.array(PIL.Image.fromarray(img).resize((size, size), resample=PIL.Image.BILINEAR))


def _is_open(task, zoom=None):
    if task.status != 'unfinished' or task.submitted:
        return False
    return zoom is None or task.cur_zoom == zoom


def _is_fresh(task):
    return (task.status == 'unfinished' and task.result == 'unknown' and not task.submitted and task.cur_zoom_idx == 0
            and task.cur_iter == 0 and task.total_iter == 0 and len(task.loc_history) == 1 and not task.job_history
            and not task.all_loc_to_dict and not task.loc_to_at_zoom)


def _exact_point(p):
    """An (x, y) array whose arithmetic in RefinementTask is fp64 arithmetic on its values: float64 and finite, float32
    below 2**24 in magnitude, or integers that fp64 holds exactly (Python raises on NaN / inf positions).
    float32: `pos - size // 2` and `loc - patch.x` are exact in fp32 where the crop is not clamped (a multiple of ulp(pos)
    no larger than pos), and an fp64 quotient rounded to fp32 equals the fp32 quotient (53 >= 2 * 24 + 2)."""
    if not (isinstance(p, np.ndarray) and p.shape == (2,)):
        return False
    if p.dtype == np.float64:
        return bool(np.isfinite(p).all())
    if p.dtype == np.float32:
        return bool((np.abs(p) < 2.0 ** 24).all())
    return p.dtype.kind in 'iu' and bool((np.abs(p.astype(np.float64)) < 2.0 ** 52).all())


def _submit_rect(t, rect):
    """RefinementTask._submit of a job whose crops are `rect` [x_from, y_from, size_from, x_to, y_to, size_to] (its own or
    its pilot's), with the device-pixel paths' 'img' key."""
    x0, y0, s0, x1, y1, s1 = (int(v) for v in rect)
    (h_f, w_f), (h_t, w_t) = t.image_from.shape[:2], t.image_to.shape[:2]
    t.cur_job = {'patch_from': ImagePatch(None, x0, y0, s0, s0, w_f, h_f), 'patch_to': ImagePatch(None, x1, y1, s1, s1, w_t, h_t),
                 'loc_from': t.loc_from, 'loc_to': t.cur_loc_to, 'img': None}
    t.job_history.append((s0, s0, s1, s1))


def _replay_level(t, rect, loc, good):
    """What a device walk did to task `t` at its current level, as the host loop leaves it: submit with `rect`, then
    RefinementTask.step to `loc` (fp64 (2,)) with converge_iters 1, and next_zoom; `good` decides the last level."""
    _submit_rect(t, rect)
    last = t.cur_zoom_idx == len(t.zoom_ins) - 1
    loc = loc.copy()
    t.total_iter += 1
    t.loc_to_at_zoom.append(loc)
    if last:
        t.cur_iter += 1
    t.all_loc_to_dict[t.cur_zoom] = np.array(t.loc_to_at_zoom).copy()
    t.loc_history.append(loc)
    t.best_loc_to = loc
    t.cur_loc_to = loc
    if last:
        t.status = 'finished'
        t.result = 'good' if good else 'bad'
    t.cur_zoom_idx += 1
    t.cur_iter = 0
    t.loc_to_at_zoom = []


def _rect_of(task):
    pf, pt = task.cur_job['patch_from'], task.cur_job['patch_to']
    assert pf.w == pf.h and pt.w == pt.h
    return (pf.x, pf.y, pf.w, pt.x, pt.y, pt.w)


class SparseEngine():
    def __init__(self, model, batch_size, mode='stretching', device_preprocess=True, device_walk=False):
        assert mode in ['stretching', 'tile']
        self.model = model
        self.batch_size = batch_size
        self.total_tasks = 0
        self.mode = mode
        # When the model is the native one, the crops are resized / normalised on the device (bit-identical to the
        # host PIL path, which remains the behaviour for any other model) - see COTR.preprocess_canvases.
        self.device_preprocess = device_preprocess
        # device_walk: the single-query loop runs as one device call (COTR.refine_walk) when it can; same results
        self.device_walk = device_walk
        self._dev_images = {}

    # ---- device-side pixels --------------------------------------------------------------------------------
    def _device_pixels_fit(self, images):
        """The model takes pixels on the device and every image is a uint8 HWC RGB array."""
        if not (self.device_preprocess and getattr(self.model, 'supports_device_preprocess', False)):
            return False
        try:
            if next(self.model.parameters()).device.type != 'cuda':
                return False
        except StopIteration:
            return False
        return all(isinstance(img, np.ndarray) and img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3 for img in images)

    def _use_device_pixels(self, tasks):
        first = tasks[0]
        if not self._device_pixels_fit((first.image_from, first.image_to)):
            return False
        return all(t.image_from is first.image_from and t.image_to is first.image_to for t in tasks)

    def _device_stretch(self, img_a, img_b):
        """'stretching' mode's stretch, dense pass and resize back run on the device (stretched_flow_maps)."""
        return (inference_helper.DEVICE_STRETCH and hasattr(self.model, 'resize_image') and hasattr(self.model, 'resize_maps')
                and self._device_pixels_fit((img_a, img_b)) and flow_on_device(self.model, img_a, img_b))

    def _device_image(self, img):
        key = (id(img), img.shape)
        hit = self._dev_images.get(key)
        if hit is None or hit[0] is not img:
            if len(self._dev_images) > 8:
                self._dev_images.clear()
            dev = next(self.model.parameters()).device
            hit = (img, torch.from_numpy(np.ascontiguousarray(img)).to(dev))
            self._dev_images[key] = hit
        return hit[1]

    def _device_canvases(self, tasks):
        rects = np.array([_rect_of(t) for t in tasks], dtype=np.int32)
        return self.model.preprocess_canvases(self._device_image(tasks[0].image_from), self._device_image(tasks[0].image_to), rects)

    # ---- batching ------------------------------------------------------------------------------------------
    def form_batch(self, tasks, zoom=None, start=0):
        """First `batch_size` open tasks (optionally at one zoom level) -> stacked canvases and queries (:25-45).
        `start`: the caller knows that no task before this index is open (the scan is the same, only shorter)."""
        chosen = []
        for i in range(start, len(tasks)):
            t = tasks[i]
            if _is_open(t, zoom):
                chosen.append(t)
                if len(chosen) >= self.batch_size:
                    break
        if not chosen:
            return [], [], []
        if self._use_device_pixels(chosen):
            queries = [t.get_task_fast()[1] for t in chosen]           # geometry + query only
            return chosen, self._device_canvases(chosen), torch.stack(queries)
        imgs, queries = [], []
        for t in chosen:
            img, query = t.get_task()
            imgs.append(img)
            queries.append(query)
        return chosen, torch.stack(imgs), torch.stack(queries)

    def infer_batch(self, img_batch, query_batch):
        """(n,3,256,512) + (n,1,2) -> (n,2) numpy; NaN raises like the reference (:47-56)."""
        self.total_tasks += img_batch.shape[0]
        device = next(self.model.parameters()).device
        out = self.model(img_batch.to(device), query_batch.to(device))['pred_corrs'].clone().detach()
        out = out.cpu().numpy()[:, 0, :]
        if utils.has_nan(out):
            raise ValueError('NaN in prediction')
        return out

    def conclude_tasks(self, tasks, return_idx=False, force=False, offset_x_from=0, offset_y_from=0, offset_x_to=0,
                       offset_y_to=0, img_a_shape=None, img_b_shape=None):
        """Collect accepted results of finished tasks; drop those on / outside the image borders (:58-84)."""
        corrs, idx = [], []
        for t in tasks:
            if t.status != 'finished':
                continue
            out = t.conclude(force)
            if out is not None:
                corrs.append(np.array(out))
                idx.append(t.identifier)
        corrs = np.array(corrs)
        idx = np.array(idx)
        if corrs.shape[0] > 0:
            corrs -= np.array([offset_x_from, offset_y_from, offset_x_to, offset_y_to])
            if img_a_shape is not None and img_b_shape is not None and not force:
                upper = np.concatenate([img_a_shape[::-1], img_b_shape[::-1]])
                inside = np.all(corrs < upper, axis=1) & np.all(corrs > 0, axis=1)
                corrs = corrs[inside]
                idx = idx[inside]
        if return_idx:
            return corrs, idx
        return corrs

    def num_finished_tasks(self, tasks):
        return sum(1 for t in tasks if t.status == 'finished')

    def num_good_tasks(self, tasks):
        return sum(1 for t in tasks if t.result == 'good')

    # ---- task generation -----------------------------------------------------------------------------------
    def gen_tasks_w_known_scale(self, img_a, img_b, queries_a, areas, zoom_ins=[1.0], converge_iters=1, max_corrs=1000):
        assert self.mode == 'tile'
        corr_a = cotr_corr_base(self.model, img_a, img_b, queries_a)
        return [RefinementTask(img_a, img_b, c[:2], c[2:], areas[0], areas[1], converge_iters, zoom_ins) for c in corr_a]

    def _dense_first_guess(self, img_a, img_b):
        """cotr_flow's maps on the pair (stretched to squares in 'stretching' mode, :114-139) as
        (corr_a, con_a, None, corr_b, con_b, None): the warped images cotr_flow also returns are never used here, so they
        are not computed.  The maps are float64, except after a stretch, where float_image_resize leaves them float32
        (which changes gen_tasks' arithmetic: its compares and first guesses then run in float32).  With the native model
        the stretch, the dense pass and the resize back run on the device, and only the four maps come to the host."""
        needs_stretch = self.mode == 'stretching' and (img_a.shape[0] != img_a.shape[1] or img_b.shape[0] != img_b.shape[1])
        if self.mode not in ('stretching', 'tile'):
            raise ValueError(f'unsupported mode: {self.mode}')
        if not needs_stretch:
            corr_a, con_a, corr_b, con_b = cotr_flow_maps(self.model, img_a, img_b)
            return corr_a, con_a, None, corr_b, con_b, None
        shape_a, shape_b = img_a.shape[:2], img_b.shape[:2]
        if self._device_stretch(img_a, img_b):
            (corr_a, con_a), (corr_b, con_b) = stretched_flow_maps(self.model, self._device_image(img_a), self._device_image(img_b),
                                                                   shape_a, shape_b)
            return corr_a.cpu().numpy(), con_a.cpu().numpy(), None, corr_b.cpu().numpy(), con_b.cpu().numpy(), None
        corr_a, con_a, corr_b, con_b = cotr_flow_maps(self.model, stretch_to_square_np(img_a.copy()), stretch_to_square_np(img_b.copy()))
        resize = utils.float_image_resize
        return resize(corr_a, shape_a), resize(con_a, shape_a), None, resize(corr_b, shape_b), resize(con_b, shape_b), None

    def gen_tasks(self, img_a, img_b, zoom_ins=[1.0], converge_iters=1, max_corrs=1000, queries_a=None, force=False, areas=None):
        if areas is not None:
            assert queries_a is not None
            assert force == True
            assert max_corrs >= queries_a.shape[0]
            return self.gen_tasks_w_known_scale(img_a, img_b, queries_a, areas, zoom_ins=zoom_ins,
                                                converge_iters=converge_iters, max_corrs=max_corrs)
        corr_a, con_a, _, corr_b, con_b, _ = self._dense_first_guess(img_a, img_b)
        mask_a = con_a < THRESHOLD_SPARSE
        mask_b = con_b < THRESHOLD_SPARSE
        area_a = (con_a < THRESHOLD_AREA).sum() / mask_a.size
        area_b = (con_b < THRESHOLD_AREA).sum() / mask_b.size
        size_a_xy = img_a.shape[:2][::-1]
        size_b_xy = img_b.shape[:2][::-1]

        def guess(corr, pos_rc, size_xy):
            """[-1,1] dense prediction at integer pixel (row, col) -> pixel location in the other image."""
            return (corr[tuple(pos_rc)].copy() * 0.5 + 0.5) * size_xy

        def new_task(loc_from, loc_to, identifier=None):
            return RefinementTask(img_a, img_b, loc_from, loc_to, area_a, area_b, converge_iters, zoom_ins, identifier=identifier)

        tasks = []
        if queries_a is None:
            # sample (with replacement) confident pixels of both dense maps (:147-166); RNG order: a then b
            cand_a = np.array(np.where(mask_a)).T
            cand_a = cand_a[np.random.choice(len(cand_a), min(max_corrs, len(cand_a)))]
            cand_b = np.array(np.where(mask_b)).T
            cand_b = cand_b[np.random.choice(len(cand_b), min(max_corrs, len(cand_b)))]
            for pos in cand_a:
                tasks.append(new_task(pos[::-1], guess(corr_a, np.floor(pos).astype('int'), size_b_xy)))
            for pos in cand_b:
                # b->a samples keep their first guess as the fixed end: from/to are swapped on purpose (:159-166)
                tasks.append(new_task(guess(corr_b, np.floor(pos).astype('int'), size_a_xy), pos[::-1]))
            return tasks

        if force:
            for i, loc_from in enumerate(queries_a):
                pos = loc_from[::-1]
                pos = np.array([np.clip(pos[0], 0, corr_a.shape[0] - 1), np.clip(pos[1], 0, corr_a.shape[1] - 1)], dtype=int)
                tasks.append(new_task(loc_from, guess(corr_a, pos, size_b_xy), identifier=i))
            return tasks

        def usable(loc_from):
            pos = loc_from[::-1]
            if (pos > np.array(img_a.shape[:2]) - 1).any() or (pos < 0).any():
                return None
            return np.floor(pos).astype('int')

        for i, loc_from in enumerate(queries_a):          # confident queries first (:176-182)
            pos = usable(loc_from)
            if pos is not None and mask_a[tuple(pos)]:
                tasks.append(new_task(loc_from, guess(corr_a, pos, size_b_xy), identifier=i))
        if len(tasks) < max_corrs:                        # then top up with unconfident ones (:183-195)
            extra = max_corrs - len(tasks)
            added = 0
            for i, loc_from in enumerate(queries_a):
                if added >= extra:
                    break
                pos = usable(loc_from)
                if pos is not None and mask_a[tuple(pos)] == False:
                    tasks.append(new_task(loc_from, guess(corr_a, pos, size_b_xy), identifier=i))
                    added += 1
        return tasks

    # ---- drivers -------------------------------------------------------------------------------------------
    def _single_query_loop(self, tasks, max_corrs, zoom=None):
        """The reference rescans every task three times per batch (good / finished counts for its progress line and the
        first-open search, :201-211, :25-45): quadratic in the task count.  Same decisions and the same printed lines here
        from running counts and a cursor - inside this loop only the tasks of the current batch change state, and a
        task that is not open (finished, already submitted, or at another zoom level) cannot become open again."""
        if self.device_walk and zoom is None and self._device_walk_fits(tasks):
            self._device_walk(tasks, max_corrs)
            return
        num_g, num_f, start = self.num_good_tasks(tasks), self.num_finished_tasks(tasks), 0
        while True:
            print(f'{num_g} / {max_corrs} | {num_f} / {len(tasks)}')
            while start < len(tasks) and not _is_open(tasks[start], zoom):
                start += 1
            task_ref, img_batch, query_batch = self.form_batch(tasks, zoom, start)
            if len(task_ref) == 0 or num_g >= max_corrs:
                break
            out = self.infer_batch(img_batch, query_batch)
            for t, o in zip(task_ref, out):
                t.step(o)
                if t.status == 'finished':
                    num_f += 1
                    num_g += t.result == 'good'

    def _device_walk_fits(self, tasks):
        return hasattr(self.model, 'refine_walk') and self._walk_fits(tasks)

    def _walk_fits(self, tasks):
        """The device walks' conditions: device pixels, fresh tasks with converge_iters 1, one (s_from, s_to) and one zoom
        schedule of <= 7 levels, and every crop at least 2 pixels wide (anything else raises in the host loop too)."""
        if not tasks or not self._use_device_pixels(tasks):
            return False
        first = tasks[0]
        zooms = list(first.zoom_ins)
        if not 1 <= len(zooms) <= 7:
            return False
        for t in tasks:
            if not (t.converge_iters == 1 and _is_fresh(t) and t.s_from == first.s_from and t.s_to == first.s_to
                    and (t.zoom_ins is first.zoom_ins or list(t.zoom_ins) == zooms)
                    and _exact_point(t.loc_from) and _exact_point(t.cur_loc_to)):
                return False
        for z in zooms:
            for s, img in ((first.s_from, first.image_from), (first.s_to, first.image_to)):
                scale = s * z
                if scale != scale or get_patch_centered_at(None, (0, 0), scale, False, img.shape).w < 2:
                    return False
        return True

    def _device_walk(self, tasks, max_corrs):
        """_single_query_loop as one COTR.refine_walk call; every walked task is left exactly as the host loop leaves it,
        and the same progress lines are printed."""
        first = tasks[0]
        n, L, batch = len(tasks), len(first.zoom_ins), self.batch_size
        max_good = math.ceil(max_corrs) if max_corrs <= n else n
        image_from, image_to = self._device_image(first.image_from), self._device_image(first.image_to)
        history, rects, good, walked, (code, chunk, level) = self.model.refine_walk(
            [image_from, image_to], [(0, 1, 0, n, float(first.s_from), float(first.s_to))], [float(z) for z in first.zoom_ins],
            batch, max_good, refinement_task.THRESHOLD_PIXELS_RELATIVE, [t.loc_from for t in tasks], [t.cur_loc_to for t in tasks])
        num_g = num_f = 0
        for c0 in range(0, walked, batch):
            for _ in range(L):
                print(f'{num_g} / {max_corrs} | {num_f} / {n}')
            c1 = min(c0 + batch, n)
            num_g += int(good[c0:c1].sum())
            num_f += c1 - c0
        self.total_tasks += walked * L
        if code != 0:
            for _ in range(level + 1):
                print(f'{num_g} / {max_corrs} | {num_f} / {n}')
            self.total_tasks += (min(walked + batch, n) - walked) * (level + 1)
            raise ValueError('NaN in prediction' if code == 1 else 'non-finite position in the zoom-in walk')
        print(f'{num_g} / {max_corrs} | {num_f} / {n}')
        for i in range(walked):
            for l in range(L):
                _replay_level(tasks[i], rects[i, l], history[i, l + 1], l == L - 1 and bool(good[i]))
        # the host loop forms (submits) the next batch before it tests max_corrs and stops
        for t in tasks[walked:walked + batch]:
            t.get_task_fast()

    def _finish(self, tasks, max_corrs, return_idx, force, return_tasks_only, img_a_shape, img_b_shape):
        if return_tasks_only:
            return tasks
        if return_idx:
            corrs, idx = self.conclude_tasks(tasks, return_idx=True, force=force, img_a_shape=img_a_shape, img_b_shape=img_b_shape)
            return corrs[:max_corrs], idx[:max_corrs]
        return self.conclude_tasks(tasks, force=force, img_a_shape=img_a_shape, img_b_shape=img_b_shape)[:max_corrs]

    def cotr_corr_multiscale(self, img_a, img_b, zoom_ins=[1.0], converge_iters=1, max_corrs=1000, queries_a=None,
                             return_idx=False, force=False, return_tasks_only=False, areas=None):
        """Correspondences (<=max_corrs, 4) [x_a, y_a, x_b, y_b] in pixels (:197-233)."""
        img_a = img_a.copy()
        img_b = img_b.copy()
        if queries_a is not None:
            queries_a = queries_a.copy()
        tasks = self.gen_tasks(img_a, img_b, zoom_ins, converge_iters, max_corrs, queries_a, force, areas)
        self._single_query_loop(tasks, max_corrs)
        return self._finish(tasks, max_corrs, return_idx, force, return_tasks_only, img_a.shape[:2], img_b.shape[:2])

    def cotr_corr_multiscale_with_cycle_consistency(self, img_a, img_b, zoom_ins=[1.0], converge_iters=1, max_corrs=1000,
                                                    queries_a=None, return_idx=False, return_cycle_error=False):
        """a->b, then b->a on the a->b answers; keep the max_corrs smallest cycle errors (:235-264)."""
        EXTRACTION_RATE = 0.3
        temp_max_corrs = int(max_corrs / EXTRACTION_RATE)
        if queries_a is not None:
            temp_max_corrs = min(temp_max_corrs, queries_a.shape[0])
            queries_a = queries_a.copy()
        corr_f, idx_f = self.cotr_corr_multiscale(img_a.copy(), img_b.copy(), zoom_ins=zoom_ins, converge_iters=converge_iters,
                                                  max_corrs=temp_max_corrs, queries_a=queries_a, return_idx=True)
        assert corr_f.shape[0] > 0
        corr_b, idx_b = self.cotr_corr_multiscale(img_b.copy(), img_a.copy(), zoom_ins=zoom_ins, converge_iters=converge_iters,
                                                  max_corrs=corr_f.shape[0], queries_a=corr_f[:, 2:].copy(), return_idx=True)
        assert corr_b.shape[0] > 0
        cycle_errors = np.linalg.norm(corr_f[idx_b][:, :2] - corr_b[:, 2:], axis=1)
        order = np.argsort(cycle_errors)
        out = [corr_f[idx_b][order][:max_corrs]]
        if return_idx:
            out.append(idx_f[idx_b][order][:max_corrs])
        if return_cycle_error:
            out.append(cycle_errors[order][:max_corrs])
        return out[0] if len(out) == 1 else out


class FasterSparseEngine(SparseEngine):
    """Nearby tasks share one network context: faster, slightly less accurate (:267-427).

    `rescue_stranded` (default False = the reference's behaviour) finishes, one query per context, the tasks the
    reference silently drops: a zoom level stops grouping as soon as one invocation solves <= batch_size sub-tasks
    (:398-399), and the single-query fallback only picks up tasks sitting at the LAST zoom value (:401-411), so tasks
    left behind at an earlier level never reach 'finished' (SURVEY.md section 3.3).
    """

    def __init__(self, model, batch_size, mode='stretching', max_load=256, device_preprocess=True, rescue_stranded=False,
                 device_grouping=True, device_walk=False):
        super().__init__(model, batch_size, mode=mode, device_preprocess=device_preprocess, device_walk=device_walk)
        self.max_load = max_load
        self.rescue_stranded = rescue_stranded
        # squads are formed on the device (cotr_group_tasks) whenever the pixels are made there too; the result is
        # identical to the host walk of form_squad (same order, same strict float64 comparisons)
        self.device_grouping = device_grouping
        self._squad_pixels_on_device = False

    def infer_batch_grouped(self, img_batch, query_batch):
        device = next(self.model.parameters()).device
        return self.model(img_batch.to(device), query_batch.to(device))['pred_corrs'].clone().detach().cpu().numpy()

    def get_tasks_map(self, zoom, tasks):
        """(n,4) [x_from, y_from, x_to, y_to] of every open task at `zoom` + their indices into `tasks` (:284-293)."""
        points, ids = [], []
        for i, t in enumerate(tasks):
            if _is_open(t, zoom):
                # what peek() reports as loc_from / loc_to (refinement_task.py:59-69) without building its two patches
                points.append(np.concatenate([t.loc_from, t.cur_loc_to]))
                ids.append(i)
        return np.array(points), np.array(ids)

    def form_squad(self, zoom, pilot, pilot_id, tasks, tasks_map, task_ids, bookkeeping):
        """The pilot's crops define the context; free tasks whose two end points fall in the central half of both
        crops ride along (at most max_load of them) (:295-337)."""
        assert pilot.status == 'unfinished' and pilot.submitted == False and pilot.cur_zoom == zoom
        SAFE_AREA = 0.5
        info = pilot.peek()

        def safe_box(p):
            cx, cy = p.x + p.w / 2, p.y + p.h / 2
            return cx - p.w / 2 * SAFE_AREA, cx + p.w / 2 * SAFE_AREA, cy - p.h / 2 * SAFE_AREA, cy + p.h / 2 * SAFE_AREA

        f_l, f_r, f_u, f_d = safe_box(info['patch_from'])
        t_l, t_r, t_u, t_d = safe_box(info['patch_to'])
        img, query = pilot.get_task_fast() if self._squad_pixels_on_device else pilot.get_task()
        assert pilot.submitted == True
        members, queries = [pilot], [query]
        bookkeeping[pilot_id] = False
        fits = ((tasks_map[:, 0] > f_l) & (tasks_map[:, 0] < f_r) & (tasks_map[:, 1] > f_u) & (tasks_map[:, 1] < f_d) &
                (tasks_map[:, 2] > t_l) & (tasks_map[:, 2] < t_r) & (tasks_map[:, 3] > t_u) & (tasks_map[:, 3] < t_d))
        loads = np.where(fits * bookkeeping)[0][: self.max_load]
        for ti in task_ids[loads]:
            t = tasks[ti]
            assert t.status == 'unfinished' and t.submitted == False and t.cur_zoom == zoom
            _, query = t.get_task_pilot(pilot)
            members.append(t)
            queries.append(query)
        bookkeeping[loads] = False
        return members, img, torch.stack(queries, axis=1), bookkeeping

    @staticmethod
    def _pilot_boxes(candidates):
        """(n,8) [f_l, f_r, f_u, f_d, t_l, t_r, t_u, t_d]: the central-half boxes (SAFE_AREA of form_squad) of the crops
        every candidate would use as a pilot - `get_patch_centered_at` (inference_helper.py:78-102) vectorised over the
        tasks with the same float64 expressions and the same int() truncations."""
        first = candidates[0]
        out = np.empty((len(candidates), 8), dtype=np.float64)
        sides = ((0, np.array([c.loc_from for c in candidates], dtype=np.float64), np.array([c.s_from * c.cur_zoom for c in candidates]), first.image_from.shape),
                 (4, np.array([c.cur_loc_to for c in candidates], dtype=np.float64), np.array([c.s_to * c.cur_zoom for c in candidates]), first.image_to.shape))
        for col, pos, scale, shape in sides:
            h, w = shape[0], shape[1]
            size = min(h, w) * np.clip(scale, 0.0, 1.0)
            size = ((size // 2) * 2).astype(np.int64)
            top = np.trunc(pos[:, 1] - size // 2).astype(np.int64)
            left = np.trunc(pos[:, 0] - size // 2).astype(np.int64)
            top = np.maximum(top, 0)
            left = np.maximum(left, 0)
            top = np.where(top + size > h, h - size, top)
            left = np.where(left + size > w, w - size, left)
            cx, cy = left + size / 2, top + size / 2
            out[:, col + 0] = cx - size / 2 * 0.5
            out[:, col + 1] = cx + size / 2 * 0.5
            out[:, col + 2] = cy - size / 2 * 0.5
            out[:, col + 3] = cy + size / 2 * 0.5
        return out

    def _form_squads_on_device(self, zoom, tasks, tasks_map, task_ids):
        """form_squad for the whole batch in one device call (cotr_group_tasks); the per-task bookkeeping (`submitted`,
        `cur_job`, the queries in the pilot's frame) is then replayed on the host in the reference's order."""
        from .. import capi
        candidates = [tasks[ti] for ti in task_ids]
        boxes = self._pilot_boxes(candidates)
        device = next(self.model.parameters()).device
        squad, rank, n_squads = capi.group_tasks(tasks_map, boxes, self.batch_size, self.max_load, device)
        task_ref, queries = [], []
        order = np.lexsort((rank, squad))
        order = order[squad[order] >= 0]
        bounds = np.searchsorted(squad[order], np.arange(n_squads + 1))
        for s in range(n_squads):
            idx = order[bounds[s]:bounds[s + 1]]
            pilot = candidates[idx[0]]
            assert pilot.status == 'unfinished' and pilot.submitted == False and pilot.cur_zoom == zoom
            _, query = pilot.get_task_fast()
            members, qs = [pilot], [query]
            for i in idx[1:]:
                t = candidates[i]
                assert t.status == 'unfinished' and t.submitted == False and t.cur_zoom == zoom
                _, query = t.get_task_pilot(pilot)
                members.append(t)
                qs.append(query)
            task_ref.append(members)
            queries.append(torch.stack(qs, axis=1))
        return task_ref, queries

    def form_grouped_batch(self, zoom, tasks):
        """Up to batch_size squads; queries zero-padded to the longest squad (:339-369)."""
        tasks_map, task_ids = self.get_tasks_map(zoom, tasks)
        candidates = [tasks[i] for i in task_ids] if len(task_ids) else []
        self._squad_pixels_on_device = bool(candidates) and self._use_device_pixels(candidates)
        shuffle = np.random.permutation(tasks_map.shape[0])
        tasks_map = np.take(tasks_map, shuffle, axis=0)
        task_ids = np.take(task_ids, shuffle, axis=0)
        if self._squad_pixels_on_device and self.device_grouping:
            task_ref, queries = self._form_squads_on_device(zoom, tasks, tasks_map, task_ids)
            if not task_ref:
                return [], [], []
            longest = max(q.shape[1] for q in queries)
            queries = [torch.cat([q, torch.zeros([1, longest - q.shape[1], 2])], axis=1) for q in queries]
            return task_ref, self._device_canvases([squad[0] for squad in task_ref]), torch.cat(queries)
        bookkeeping = np.ones_like(task_ids).astype(bool)
        task_ref, imgs, queries = [], [], []
        for i, ti in enumerate(task_ids):
            t = tasks[ti]
            if not _is_open(t, zoom):
                continue
            members, img, q, bookkeeping = self.form_squad(zoom, t, i, tasks, tasks_map, task_ids, bookkeeping)
            task_ref.append(members)
            imgs.append(img)
            queries.append(q)
            if len(task_ref) >= self.batch_size:
                break
        if not task_ref:
            return [], [], []
        longest = max(q.shape[1] for q in queries)
        queries = [torch.cat([q, torch.zeros([1, longest - q.shape[1], 2])], axis=1) for q in queries]
        if self._squad_pixels_on_device:
            img_batch = self._device_canvases([squad[0] for squad in task_ref])      # one context per pilot
        else:
            img_batch = torch.stack(imgs)
        return task_ref, img_batch, torch.cat(queries)

    def _grouped_walk_fits(self, tasks, zoom_ins):
        """The device walk of the grouped levels applies: the single-query walk's conditions, device grouping, no attention
        hooks (the host loop fires them per batch), pairwise distinct zoom values (with a repeated one `_is_open` matches
        tasks of two levels and all_loc_to_dict merges them), and float64 end points in get_tasks_map (float32 points
        on both ends would be compared in float32 there)."""
        if not (self.device_walk and self.device_grouping and hasattr(self.model, 'refine_grouped_batch')):
            return False
        if not (isinstance(self.batch_size, int) and self.batch_size >= 1 and isinstance(self.max_load, int) and self.max_load >= 0):
            return False
        if self.model.attention_hooked() or not self._walk_fits(tasks):
            return False
        zooms = [float(z) for z in tasks[0].zoom_ins]
        if len(set(zooms)) != len(zooms) or [float(z) for z in zoom_ins] != zooms:
            return False
        return np.result_type(*{a.dtype for t in tasks for a in (t.loc_from, t.cur_loc_to)}) == np.float64

    def _grouped_walk(self, tasks, zoom_ins, max_corrs):
        """The `for zm in zoom_ins` loop of cotr_corr_multiscale with one COTR.refine_grouped_batch call per grouped batch:
        the same np.random.permutation calls, printed lines and task attributes as the host loop.  The host keeps each
        level's open tasks (those stepped at the level before and not yet taken) in index order."""
        first = tasks[0]
        n, L = len(tasks), len(first.zoom_ins)
        dev = next(self.model.parameters()).device
        image_from, image_to = self._device_image(first.image_from), self._device_image(first.image_to)
        history = torch.zeros((n, L + 1, 2), dtype=torch.float64)
        history[:, 0] = torch.from_numpy(np.array([t.cur_loc_to for t in tasks], dtype=np.float64))
        walk = {'loc_from': torch.from_numpy(np.array([t.loc_from for t in tasks], dtype=np.float64)).to(dev),
                'history': history.to(dev), 'rects': torch.zeros((n, L, 6), dtype=torch.int32, device=dev),
                'good': torch.zeros(n + 1, dtype=torch.int32, device=dev)}
        # num_g >= max_corrs, with num_g counting the good tasks on the device (NaN max_corrs never stops)
        max_good = math.ceil(max_corrs) if max_corrs <= n else n + 1
        steps = np.zeros(n, dtype=np.int64)             # levels each task was stepped at
        submitted = np.zeros(n, dtype=bool)             # formed into a squad at the max_corrs stop, never stepped
        open_ids = np.arange(n)
        for l, zm in enumerate(zoom_ins):
            print(f'======= Zoom: {zm} ======')
            stepped = []
            while True:
                ids = np.take(open_ids, np.random.permutation(open_ids.shape[0]), axis=0)
                squad, (n_squads, longest, num_steps, ran, status) = self.model.refine_grouped_batch(
                    image_from, image_to, first.s_from, first.s_to, [float(z) for z in first.zoom_ins], l, ids, self.batch_size,
                    self.max_load, max_good, refinement_task.THRESHOLD_PIXELS_RELATIVE, walk)
                if status == 1:
                    raise ValueError('cannot convert float NaN to integer')
                if status == 2:
                    raise OverflowError('cannot convert float infinity to integer')
                if n_squads == 0:
                    break
                taken = ids[squad >= 0]
                open_ids = np.sort(ids[squad < 0])
                if not ran:
                    submitted[taken] = True
                    break
                steps[taken] += 1
                stepped.append(taken)
                print(f'solved {num_steps} sub-tasks in one invocation with {n_squads} image pairs')
                if num_steps <= self.batch_size:
                    break
            open_ids = np.sort(np.concatenate(stepped)) if stepped else np.zeros(0, dtype=np.int64)
        history = walk['history'].cpu().numpy()
        rects = walk['rects'].cpu().numpy()
        good = walk['good'].cpu().numpy()
        for i in np.flatnonzero((steps > 0) | submitted):
            t = tasks[i]
            for l in range(steps[i]):
                _replay_level(t, rects[i, l], history[i, l + 1], l == L - 1 and bool(good[i]))
            if submitted[i]:
                _submit_rect(t, rects[i, steps[i]])
                t.submitted = True

    def cotr_corr_multiscale(self, img_a, img_b, zoom_ins=[1.0], converge_iters=1, max_corrs=1000, queries_a=None,
                             return_idx=False, force=False, return_tasks_only=False, areas=None):
        img_a = img_a.copy()
        img_b = img_b.copy()
        if queries_a is not None:
            queries_a = queries_a.copy()
        tasks = self.gen_tasks(img_a, img_b, zoom_ins, converge_iters, max_corrs, queries_a, force, areas)
        if self._grouped_walk_fits(tasks, zoom_ins):
            self._grouped_walk(tasks, zoom_ins, max_corrs)
            zm = zoom_ins[-1]
        else:
            for zm in zoom_ins:
                print(f'======= Zoom: {zm} ======')
                while True:
                    num_g = self.num_good_tasks(tasks)
                    task_ref, img_batch, query_batch = self.form_grouped_batch(zm, tasks)
                    if len(task_ref) == 0 or num_g >= max_corrs:
                        break
                    out = self.infer_batch_grouped(img_batch, query_batch)
                    num_steps = 0
                    for i, squad in enumerate(task_ref):
                        for j, t in enumerate(squad):
                            t.step(out[i, j])
                            num_steps += 1
                    print(f'solved {num_steps} sub-tasks in one invocation with {img_batch.shape[0]} image pairs')
                    if num_steps <= self.batch_size:     # grouping no longer pays at this level (:398-399)
                        break
        # one-query-per-context fallback, only for tasks sitting at the LAST zoom value (:401-411)
        self._single_query_loop(tasks, max_corrs, zm)
        if self.rescue_stranded:
            self._single_query_loop(tasks, max_corrs)     # whatever is still open, at whatever level it was left
        return self._finish(tasks, max_corrs, return_idx, force, return_tasks_only, img_a.shape[:2], img_b.shape[:2])
