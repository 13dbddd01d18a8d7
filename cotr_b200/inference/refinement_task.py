"""Per-correspondence zoom-in state machine (reference: COTR/inference/refinement_task.py).

A task walks the zoom schedule: at every level it crops a patch around its source point and around the current
estimate, asks the network where the source point lands in the target patch, maps the answer back to pixels and
zooms in.  The last level repeats up to `converge_iters` times (or until the prediction revisits a value); the
estimate history decides acceptance (conclude).  Public names / attributes match the reference because the
engines and external callers poke at them (status, submitted, cur_zoom, identifier, result, loc_history ...).
"""
import numpy as np
import torch

from .inference_helper import (BASE_ZOOM, THRESHOLD_PIXELS_RELATIVE, _to_network_canvas, find_prediction_loop,
                               get_patch_centered_at)
from ..utils.utils import ImagePatch


def _geometry_only(p):
    return ImagePatch(None, p.x, p.y, p.w, p.h, p.ow, p.oh)


def crop_scales(area_from, area_to):
    """(s_from, s_to): the image with the larger co-visible area gets the larger crop (refinement_task.py:25-30).  With
    numpy float64 areas an area of 0 gives an infinite scale, and two give NaN, as in the reference."""
    if area_from < area_to:
        return BASE_ZOOM, BASE_ZOOM * np.sqrt(area_to / area_from)
    return BASE_ZOOM * np.sqrt(area_from / area_to), BASE_ZOOM


class RefinementTask():
    def __init__(self, image_from, image_to, loc_from, loc_to, area_from, area_to, converge_iters, zoom_ins, identifier=None):
        self.identifier = identifier
        self.image_from = image_from
        self.image_to = image_to
        self.loc_from = loc_from
        self.best_loc_to = loc_to
        self.cur_loc_to = loc_to
        self.area_from = area_from
        self.area_to = area_to
        self.s_from, self.s_to = crop_scales(area_from, area_to)
        self.cur_job = {}
        self.status = 'unfinished'
        self.result = 'unknown'
        self.converge_iters = converge_iters
        self.zoom_ins = zoom_ins
        self.cur_zoom_idx = 0
        self.cur_iter = 0
        self.total_iter = 0
        self.loc_to_at_zoom = []
        self.loc_history = [loc_to]
        self.all_loc_to_dict = {}
        self.job_history = []
        self.submitted = False

    @property
    def cur_zoom(self):
        return self.zoom_ins[self.cur_zoom_idx]

    @property
    def confidence_scaling_factor(self):
        if self.cur_zoom_idx > 0:
            return float(self.cur_zoom) / float(self.zoom_ins[0])
        return 1.0

    # ---- job construction ----------------------------------------------------------------------------------
    def _patches(self, with_content):
        p_from = get_patch_centered_at(self.image_from if with_content else None, self.loc_from,
                                       scale=self.s_from * self.cur_zoom, return_content=with_content,
                                       img_shape=self.image_from.shape)
        p_to = get_patch_centered_at(self.image_to if with_content else None, self.cur_loc_to,
                                     scale=self.s_to * self.cur_zoom, return_content=with_content,
                                     img_shape=self.image_to.shape)
        return p_from, p_to

    def _query_in(self, patch_from):
        # x is normalised by 2*w because the canvas is two patches wide (refinement_task.py:110)
        # the reference builds three small arrays here; the same two float64 divisions, rounded to fp32 the same way
        return torch.tensor([[(self.loc_from[0] - patch_from.x) / (patch_from.w * 2), (self.loc_from[1] - patch_from.y) / patch_from.h]],
                            dtype=torch.float32)

    def _submit(self, patch_from, patch_to, with_img_key):
        self.cur_job = {'patch_from': _geometry_only(patch_from), 'patch_to': _geometry_only(patch_to),
                        'loc_from': self.loc_from, 'loc_to': self.cur_loc_to}
        if with_img_key:
            self.cur_job['img'] = None
        self.job_history.append((patch_from.h, patch_from.w, patch_to.h, patch_to.w))
        assert self.submitted == False
        self.submitted = True

    def peek(self):
        """The patches the next job would use, without submitting it (:59-69)."""
        assert self.status == 'unfinished'
        p_from, p_to = self._patches(with_content=False)
        return {'patch_from': p_from, 'patch_to': p_to, 'loc_from': self.loc_from, 'loc_to': self.cur_loc_to}

    def get_task_pilot(self, pilot):
        """Join another task's context: express this task's source point in the pilot's patch frame (:71-85)."""
        assert self.status == 'unfinished'
        p_from = _geometry_only(pilot.cur_job['patch_from'])
        p_to = _geometry_only(pilot.cur_job['patch_to'])
        query = self._query_in(p_from)
        self._submit(p_from, p_to, with_img_key=True)
        return None, query

    def get_task_fast(self):
        """Geometry + query only, no pixels (:87-103)."""
        assert self.status == 'unfinished'
        p_from, p_to = self._patches(with_content=False)
        query = self._query_in(p_from)
        self._submit(p_from, p_to, with_img_key=True)
        return None, query

    def get_task(self):
        """Crop, resize to 256x256, normalise: (3,256,512) float32 canvas + (1,2) query (:105-132)."""
        assert self.status == 'unfinished'
        p_from, p_to = self._patches(with_content=True)
        query = self._query_in(p_from)
        img = _to_network_canvas(p_from.patch, p_to.patch)
        self._submit(p_from, p_to, with_img_key=False)
        return img, query

    # ---- state transitions -----------------------------------------------------------------------------------
    def next_zoom(self):
        if self.cur_zoom_idx >= len(self.zoom_ins) - 1:
            self.status = 'finished'
            self.result = 'bad' if self.conclude() is None else 'good'
        self.cur_zoom_idx += 1
        self.cur_iter = 0
        self.loc_to_at_zoom = []

    def scale_to_loc(self, raw_to_loc):
        """Network output (canvas-normalised, right half) -> pixel location in image_to (:145-151)."""
        raw = raw_to_loc.copy()
        patch_b = self.cur_job['patch_to']
        raw[0] = (raw[0] - 0.5) * 2
        return raw * np.array([patch_b.w, patch_b.h]) + np.array([patch_b.x, patch_b.y])

    def step(self, raw_to_loc):
        assert self.submitted == True
        self.submitted = False
        loc_to = self.scale_to_loc(raw_to_loc)
        self.total_iter += 1
        self.loc_to_at_zoom.append(loc_to)
        self.cur_loc_to = loc_to
        if self.cur_zoom_idx == len(self.zoom_ins) - 1:
            # last level: iterate until the prediction repeats itself or the budget is spent (:161-167)
            done = False
            if len(self.loc_to_at_zoom) >= 2:
                done = np.prod(self.loc_to_at_zoom[:-1] == loc_to, axis=1, keepdims=True).any()
            if self.cur_iter >= self.converge_iters - 1:
                done = True
            self.cur_iter += 1
        else:
            done = True
        if not done:
            return
        level = np.array(self.loc_to_at_zoom).copy()
        self.all_loc_to_dict[self.cur_zoom] = level
        if len(level) >= 2 and np.prod(level[:-1] == level[-1], axis=1, keepdims=True).any():
            loc_to = find_prediction_loop(level).mean(axis=0)     # average over the limit cycle (:173-178)
        self.loc_history.append(loc_to)
        self.best_loc_to = loc_to
        self.cur_loc_to = loc_to
        self.next_zoom()

    def conclude(self, force=False):
        """[x_from, y_from, x_to, y_to] or None when the estimates wandered too much across levels (:184-188)."""
        history = np.array(self.loc_history)
        if (force == False) and (max(history.std(axis=0)) >= THRESHOLD_PIXELS_RELATIVE * max(*self.image_to.shape)):
            return None
        return np.concatenate([self.loc_from, self.best_loc_to])

    def conclude_intermedia(self):
        return np.concatenate([np.array(self.loc_history), np.array(self.job_history)], axis=1)
