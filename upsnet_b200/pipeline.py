"""Pipelined serving front end for the static engine: host image in, host results out, with the PCIe copies of
neighbouring images overlapped with the compute of the current one.

The reference's test loop (`upsnet_end2end_test.py:170-200`) is strictly serial per image: H2D of the batch, forward,
`.cpu()` of the outputs.  Here three streams run concurrently:

    h2d stream      image i+1  pinned host -> device staging buffer
    compute stream  image i    staging -> the CUDA graph's input, graph replay, outputs -> device staging
    d2h stream      image i-1  device staging -> pinned host result buffers

Each direction has `depth` (default 2) staging slots guarded by CUDA events; nothing blocks the host except
`result(ticket)`, which waits for that image's D2H.  Results are the same tensors `resnet_upsnet.forward` returns
(label maps int64 like the reference's argmax), sliced to the device-side counts on the host.
"""
import numpy as np
import torch


class PipelinedEngine:
    RESULT_KEYS = ("panoptic_outputs", "fcn_outputs", "pred_boxes", "cls_probs", "cls_inds", "counts", "keep", "p_cls",
                   "p_scores", "trunc_flags")

    PIXEL_MEANS = (102.9801, 115.9465, 122.7717)     # config.network.pixel_means (BGR, caffe models)

    def __init__(self, model, im_info, depth=2, with_masks=False, with_unified=False, stuff_area_limit=4 * 64 * 64,
                 pixel_means=None, im_scale=1.0, lanes=None, label_maps=True, restore_size=False, with_combined=False,
                 combined_score_threshold=0.6, combined_fraction_threshold=0.7):
        """with_unified: also run get_unified_pan_result on the device (base_dataset.py:332-371) and return its uint8
        [H,W,3] map as 'pan_2ch'.  submit() also accepts the RAW uint8 [h,w,3] BGR image (pinned): mean subtraction,
        resize by im_scale and padding (prep_im_for_blob / im_list_to_blob) then run on the device after a 4x smaller H2D.
        restore_size: crop the two label maps to im_info[:2] and resize them back to the original image size
        (upsnet_end2end_test.py:259-266, one label_restore launch) before they are returned and before pan_2ch is
        computed from them, as the reference does before its PQ evaluation; needed whenever im_info's scale != 1 or
        the network input is padded.
        with_combined: also build the combined panoptic map (base_dataset.py:373-449 get_combined_pan_result, the
        instance output merged with the semantic head) on the device and return it as 'pan_2ch_combined'.  It does what
        the test script's im_detect + im_post + the merge do: pred_boxes[:, 1:] / im_info[2] in fp32, the masks' run
        lengths at round(im_info[:2] / im_info[2]) (upsnet_im_post_rle), then upsnet_combined_pan_result on the restored
        semantic map.  Needs restore_size=True and an im_info whose im_post size equals the restored size."""
        self.model, self.depth = model, depth
        # engine lanes: slot i computes on lane i % lanes (own CUDA-graph instance, activation pool, scratch, stream), so the
        # forward passes of `lanes` consecutive images overlap on the GPU; lanes=1 is the strictly serial compute of round 1
        self.lanes = depth if lanes is None else max(1, min(int(lanes), depth))
        self.im_info = np.asarray(im_info, dtype=np.float32).reshape(-1, 3)[0]
        self.keys = self.RESULT_KEYS + (("mask_probs",) if with_masks else ()) + (("pan_2ch",) if with_unified else ()) + \
            (("pan_2ch_combined",) if with_combined else ())
        if not label_maps:      # serving format: the unified 2-channel map replaces the two int64 label maps on the way out
            assert with_unified, "label_maps=False needs with_unified=True (pan_2ch carries class and instance id)"
            self.keys = tuple(k for k in self.keys if k not in ("panoptic_outputs", "fcn_outputs"))
        self.with_unified, self.stuff_area_limit, self.restore_size = with_unified, stuff_area_limit, restore_size
        self.pixel_means, self.im_scale = (pixel_means or self.PIXEL_MEANS), float(im_scale)
        self.with_combined = with_combined
        if with_combined:
            from . import operators as ops
            if not restore_size:
                raise ValueError("with_combined needs restore_size=True: the merge runs on the restored semantic map")
            # upsnet_end2end_test.py passes np.round(im_info[:2] / im_info[2]) to im_post, while the restore follows cv2's
            # dsize rule; the reference fails to broadcast where the two differ
            self.combined_size = tuple(int(v) for v in np.round(self.im_info[:2] / self.im_info[2]))
            restored = ops.label_restore_geometry(self.im_info)[3:]
            if self.combined_size != restored:
                raise ValueError("im_post size %s != restored label size %s for im_info %s"
                                 % (self.combined_size, restored, self.im_info.tolist()))
            self.combined_thresholds = (float(combined_score_threshold), float(combined_fraction_threshold))
        self.dev = None
        self._t = 0
        self._slots = None

    def _setup(self, host_image):
        model = self.model
        if not model._prepared:
            model.prepare()
        assert model.static_engine, "the pipelined front end drives the static (sync-free) engine"
        self.dev = next(model.parameters()).device
        assert self.dev.type == "cuda", "no CPU fallback"
        self.h2d, self.d2h = torch.cuda.Stream(self.dev), torch.cuda.Stream(self.dev)
        self.raw = host_image.dtype == torch.uint8
        if self.raw:
            from . import operators as ops
            x0, _ = ops.prep_image(host_image.to(self.dev), self.pixel_means, self.im_scale)
        else:
            x0 = torch.empty(host_image.shape, dtype=torch.float32, device=self.dev)
            x0.copy_(host_image)
        out, _ = model._run_static(x0, self.im_info)      # captures the graph on first use
        out = self._post(dict(out))
        torch.cuda.synchronize(self.dev)
        self._slots = []
        self._lane_streams = [torch.cuda.Stream(self.dev) for _ in range(self.lanes)]
        for i in range(self.depth):
            s = {"lane": i % self.lanes,
                 "in": torch.empty(host_image.shape, dtype=host_image.dtype, device=self.dev),
                 "out": {k: torch.empty_like(out[k]) for k in self.keys},
                 "host": {k: torch.empty(out[k].shape, dtype=out[k].dtype).pin_memory() for k in self.keys},
                 "in_ready": torch.cuda.Event(), "in_free": torch.cuda.Event(), "out_ready": torch.cuda.Event(),
                 "done": torch.cuda.Event()}
            s["in_free"].record(torch.cuda.current_stream(self.dev))
            s["done"].record(torch.cuda.current_stream(self.dev))
            self._slots.append(s)

    @torch.no_grad()
    def submit(self, host_image):
        """host_image: pinned fp32 [1,3,H,W] (mean-subtracted, like data['data']).  Returns a ticket."""
        if self._slots is None:
            self._setup(host_image)
        s = self._slots[self._t % self.depth]
        with torch.cuda.stream(self.h2d):
            self.h2d.wait_event(s["in_free"])              # compute has consumed this slot's previous image
            s["in"].copy_(host_image, non_blocking=True)
            s["in_ready"].record(self.h2d)
        from . import operators as ops
        lane = s["lane"]
        cur = self._lane_streams[lane]
        prev_slot = ops.WS_SLOT["i"]
        ops.WS_SLOT["i"] = lane
        try:
            with torch.cuda.stream(cur):
                cur.wait_event(s["in_ready"])
                x = s["in"]
                if self.raw:
                    x, _ = ops.prep_image(s["in"], self.pixel_means, self.im_scale)
                out, _ = self.model._run_static(x, self.im_info, lane=lane)
                out = self._post(dict(out))
                s["in_free"].record(cur)
                cur.wait_event(s["done"])                          # this slot's previous results have left the device
                for k in self.keys:
                    s["out"][k].copy_(out[k], non_blocking=True)
                s["out_ready"].record(cur)
        finally:
            ops.WS_SLOT["i"] = prev_slot
        with torch.cuda.stream(self.d2h):
            self.d2h.wait_event(s["out_ready"])
            for k in self.keys:
                s["host"][k].copy_(s["out"][k], non_blocking=True)
            s["done"].record(self.d2h)
        self._t += 1
        return self._t - 1

    def _post(self, out):
        from . import operators as ops
        if self.restore_size:
            out["fcn_outputs"], out["panoptic_outputs"] = ops.label_restore(out["fcn_outputs"], self.im_info,
                                                                            out["panoptic_outputs"])
        if self.with_unified:
            m = self.model
            out["pan_2ch"] = ops.unified_pan_result(out["fcn_outputs"], out["panoptic_outputs"], out["p_cls"][out["keep"]],
                                                    m.num_seg_classes, m.num_classes, self.stuff_area_limit,
                                                    k_dev=out["counts"][2:3], check_errors=False)
        if self.with_combined:
            m, n_dev = self.model, out["counts"][0:1]
            pb = out["pred_boxes"]
            # im_detect's pred_boxes[:, 1:] / im_info[2]: an elementwise fp32 division (a scalar divisor would be turned
            # into a multiplication by its reciprocal)
            boxes = pb[:, 1:] / torch.full((1, 1), float(self.im_info[2]), dtype=torch.float32, device=pb.device)
            rle = ops.im_post_rle(boxes, out["mask_probs"], out["cls_inds"], *self.combined_size, n_dev=n_dev)[:2]
            out["pan_2ch_combined"] = ops.combined_pan_result(out["fcn_outputs"], out["cls_probs"], out["cls_inds"], rle,
                                                              m.num_seg_classes, m.num_classes, *self.combined_thresholds,
                                                              self.stuff_area_limit, n_dev=n_dev, check_errors=False)
        return out

    def result(self, ticket):
        """Blocks until image `ticket` is on the host.  The returned tensors view this slot's pinned buffers and stay
        valid until `depth` more images have been submitted."""
        assert self._t - self.depth <= ticket < self._t, "result slot already reused (or not yet submitted)"
        s = self._slots[ticket % self.depth]
        s["done"].synchronize()
        h = s["host"]
        n1, n2, k = (int(v) for v in h["counts"].tolist())
        keep = h["keep"][:k]
        res = {"cls_probs": h["cls_probs"][:n1], "pred_boxes": h["pred_boxes"][:n1], "cls_inds": h["cls_inds"][:n1],
               "panoptic_cls_inds": h["p_cls"][:n2][keep], "panoptic_cls_probs": h["p_scores"][:n2][keep]}
        if "panoptic_outputs" in h:
            res["fcn_outputs"], res["panoptic_outputs"] = h["fcn_outputs"], h["panoptic_outputs"]
        # [detections, panoptic candidates]: != 0 when the fixed-size MaskROI buffers dropped boxes the reference keeps
        res["truncated"] = h["trunc_flags"]
        if "mask_probs" in h:
            res["mask_probs"] = h["mask_probs"][:n1]
        if "pan_2ch" in h:
            res["pan_2ch"] = h["pan_2ch"]
        if "pan_2ch_combined" in h:
            res["pan_2ch_combined"] = h["pan_2ch_combined"]
        return res

    def bytes_per_image(self):
        s = self._slots[0]
        return (s["in"].numel() * s["in"].element_size(), sum(t.numel() * t.element_size() for t in s["host"].values()))
