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

Images may differ in size.  Each image's im_info row travels to the device on the h2d stream with the image, and the
engine replays the captured graph of that image's padded shape (model._run_static keys its graphs on the input shape
only), so a dataset of mixed sizes costs one capture per padded shape and lane, not one per image.
"""
import numpy as np
import torch


class PipelinedEngine:
    RESULT_KEYS = ("panoptic_outputs", "fcn_outputs", "pred_boxes", "cls_probs", "cls_inds", "counts", "keep", "p_cls",
                   "p_scores", "trunc_flags")
    # outputs whose shape follows the image: staged in buffers sized for the largest image, returned as views
    IMAGE_KEYS = ("panoptic_outputs", "fcn_outputs", "pan_2ch", "pan_2ch_combined")

    PIXEL_MEANS = (102.9801, 115.9465, 122.7717)     # config.network.pixel_means (BGR, caffe models)

    def __init__(self, model, im_info=None, depth=2, with_masks=False, with_unified=False, stuff_area_limit=4 * 64 * 64,
                 pixel_means=None, im_scale=1.0, lanes=None, label_maps=True, restore_size=False, with_combined=False,
                 combined_score_threshold=0.6, combined_fraction_threshold=0.7, target_size=None, max_size=None,
                 max_image_shape=None, config=None, dataset=None, stride=32):
        """Two ways to build it:
          PipelinedEngine(model, im_info, ...): every image has the geometry of the row im_info [h, w, scale]; a raw
            image is resized by im_scale.  Staging buffers are sized from the first image submitted.
          PipelinedEngine(model, target_size=..., max_size=..., max_image_shape=(H, W), ...), or with config= and
            dataset= ('cityscapes' / 'coco': geometry.scale_for_test_phase reads the reference's config): each image
            gets its own geometry, the reference's test phase for its original size (geometry.image_geometry).  A raw
            image may be up to H x W; staging and pinned host buffers are sized once for that and for the largest padded
            network input target_size / max_size allow.  submit(raw) resizes and pads it on the device; submit(blob,
            im_info) takes a pre-processed fp32 blob with its row.
        with_unified: also run get_unified_pan_result on the device (base_dataset.py:332-371) and return its uint8
        [H,W,3] map as 'pan_2ch'.  submit() also accepts the RAW uint8 [h,w,3] BGR image (pinned): mean subtraction,
        resize and padding (prep_im_for_blob / im_list_to_blob) then run on the device after a 4x smaller H2D.
        restore_size: crop the two label maps to im_info[:2] and resize them back to the original image size
        (upsnet_end2end_test.py:259-266, one label_restore launch) before they are returned and before pan_2ch is
        computed from them, as the reference does before its PQ evaluation; needed whenever im_info's scale != 1 or
        the network input is padded.
        with_combined: also build the combined panoptic map (base_dataset.py:373-449 get_combined_pan_result, the
        instance output merged with the semantic head) on the device and return it as 'pan_2ch_combined'.  It does what
        the test script's im_detect + im_post + the merge do: pred_boxes[:, 1:] / im_info[2] in fp32, the masks' run
        lengths at round(im_info[:2] / im_info[2]) (upsnet_im_post_rle), then upsnet_combined_pan_result on the restored
        semantic map.  Needs restore_size=True and, per image, an im_info whose im_post size equals the restored size:
        the fixed-size form checks it at construction, the mixed-size form in submit()."""
        from .geometry import scale_for_test_phase
        self.model, self.depth = model, depth
        # engine lanes: slot i computes on lane i % lanes (own CUDA-graph instances, activation pool, scratch, stream), so
        # the forward passes of `lanes` consecutive images overlap on the GPU; lanes=1 is the strictly serial compute
        self.lanes = depth if lanes is None else max(1, min(int(lanes), depth))
        if config is not None:
            target_size, max_size = scale_for_test_phase(config, dataset)
            pixel_means = pixel_means or tuple(float(v) for v in config.network.pixel_means)
            stride = int(config.network.rpn_feat_stride[-2])
        if im_info is not None:
            if target_size is not None or max_image_shape is not None:
                raise ValueError("give either im_info (one geometry) or target_size / max_image_shape (one per image)")
            self.im_info = np.asarray(im_info, dtype=np.float32).reshape(-1, 3)[0]
            self.sizes = None
        else:
            if target_size is None or max_size is None or max_image_shape is None:
                raise ValueError("a mixed-size engine needs target_size, max_size (or config and dataset) and "
                                 "max_image_shape")
            self.im_info = None
            self.sizes = (int(target_size), int(max_size))
            self.max_image_shape = tuple(int(v) for v in max_image_shape)
        self.stride = int(stride)
        self.keys = self.RESULT_KEYS + (("mask_probs",) if with_masks else ()) + (("pan_2ch",) if with_unified else ()) + \
            (("pan_2ch_combined",) if with_combined else ())
        if not label_maps:      # serving format: the unified 2-channel map replaces the two int64 label maps on the way out
            assert with_unified, "label_maps=False needs with_unified=True (pan_2ch carries class and instance id)"
            self.keys = tuple(k for k in self.keys if k not in ("panoptic_outputs", "fcn_outputs"))
        self.with_unified, self.stuff_area_limit, self.restore_size = with_unified, stuff_area_limit, restore_size
        self.pixel_means, self.im_scale = (pixel_means or self.PIXEL_MEANS), float(im_scale)
        self.with_combined = with_combined
        if with_combined:
            if not restore_size:
                raise ValueError("with_combined needs restore_size=True: the merge runs on the restored semantic map")
            self.combined_thresholds = (float(combined_score_threshold), float(combined_fraction_threshold))
            if self.im_info is not None:
                self._geometry(self.im_info)
        self.dev = None
        self._t = 0
        self._slots = None

    def _geometry(self, im_info):
        """Host geometry of one image from its row: the restore and im_post sizes.  Raises ValueError where the
        reference's combined merge would fail to broadcast."""
        from . import operators as ops
        info = np.asarray(im_info, dtype=np.float32).reshape(-1, 3)[0].copy()
        g = {"im_info": info}
        if self.restore_size:
            g["restore"] = ops.label_restore_geometry(info)
        if self.with_combined:
            # upsnet_end2end_test.py passes np.round(im_info[:2] / im_info[2]) to im_post, while the restore follows cv2's
            # dsize rule; the reference fails to broadcast where the two differ
            g["combined_size"] = tuple(int(v) for v in np.round(info[:2] / info[2]))
            if g["combined_size"] != g["restore"][3:]:
                raise ValueError("im_post size %s != restored label size %s for im_info %s"
                                 % (g["combined_size"], g["restore"][3:], info.tolist()))
        return g

    def _image(self, host_image, im_info):
        """-> (geometry, prep scale or None, padded (Hp, Wp), label-map (h, w)) of one submitted image."""
        raw = host_image.dtype == torch.uint8
        if raw:
            h, w = int(host_image.shape[0]), int(host_image.shape[1])
            if im_info is not None:
                raise ValueError("a raw image takes its im_info from its size (mixed-size engine) or the constructor")
            if self.sizes is None:
                info, scale = self.im_info, self.im_scale
            else:
                from .geometry import image_geometry
                geo = image_geometry(h, w, *self.sizes, stride=self.stride)
                info, scale = geo.im_info, geo.scale
            ho, wo = int(np.rint(h * scale)), int(np.rint(w * scale))
            padded = (-(-ho // self.stride) * self.stride, -(-wo // self.stride) * self.stride)
        else:
            info = self.im_info if im_info is None else im_info
            if info is None:
                raise ValueError("a pre-processed blob needs its im_info row")
            scale, padded = None, (int(host_image.shape[-2]), int(host_image.shape[-1]))
        g = self._geometry(info)
        maps = g["restore"][3:] if self.restore_size else padded
        return g, scale, padded, maps

    def _capacity(self, host_image, padded, maps):
        """Staging sizes (elements): input, prepared blob, label-map pixels.  Fixed-size engine: the first image's;
        mixed-size engine: the largest image and the largest padded input its size rule allows."""
        if self.sizes is None:
            return host_image.numel(), 3 * padded[0] * padded[1], maps[0] * maps[1]
        from .geometry import image_geometry
        H, W = self.max_image_shape
        ceil = lambda v: -(-v // self.stride) * self.stride           # noqa: E731
        target, max_size = self.sizes
        pix = ceil(min(target, max_size)) * ceil(max_size)            # short side <= target, long side <= max_size
        n_in = H * W * 3 if host_image.dtype == torch.uint8 else 3 * pix
        # a restored map is the original size up to the rounding of the resize there and back: 0.5 / scale + 1 pixels,
        # and the scale only grows as the image shrinks
        e = int(np.ceil(0.5 / image_geometry(H, W, target, max_size, self.stride).scale)) + 2
        return n_in, 3 * pix, ((H + e) * (W + e) if self.restore_size else pix)

    def _setup(self, host_image, im_info):
        from . import operators as ops
        model = self.model
        if not model._prepared:
            model.prepare()
        assert model.static_engine, "the pipelined front end drives the static (sync-free) engine"
        self.dev = next(model.parameters()).device
        assert self.dev.type == "cuda", "no CPU fallback"
        self.h2d, self.d2h = torch.cuda.Stream(self.dev), torch.cuda.Stream(self.dev)
        self.raw = host_image.dtype == torch.uint8
        g, scale, padded, maps = self._image(host_image, im_info)
        n_in, n_blob, self.map_cap = self._capacity(host_image, padded, maps)
        if self.raw:
            x0, _ = ops.prep_image(host_image.to(self.dev), self.pixel_means, scale, self.stride)
        else:
            x0 = torch.empty(host_image.shape, dtype=torch.float32, device=self.dev)
            x0.copy_(host_image)
        out, _ = model._run_static(x0, g["im_info"])      # captures the graph on first use
        out = self._post(dict(out), g)
        torch.cuda.synchronize(self.dev)

        def numel(k):          # elements per label-map pixel for the image-shaped keys, else the probe's shape
            return self.map_cap * out[k].numel() // (maps[0] * maps[1]) if k in self.IMAGE_KEYS else None
        self._slots = []
        self._lane_streams = [torch.cuda.Stream(self.dev) for _ in range(self.lanes)]
        for i in range(self.depth):
            s = {"lane": i % self.lanes,
                 "in": torch.empty((n_in,), dtype=host_image.dtype, device=self.dev),
                 "x": torch.empty((n_blob,), dtype=torch.float32, device=self.dev) if self.raw else None,
                 "info": torch.empty((3,), dtype=torch.float32, device=self.dev),
                 "out": {k: torch.empty((numel(k),) if numel(k) else out[k].shape, dtype=out[k].dtype, device=self.dev)
                         for k in self.keys},
                 "host": {k: torch.empty((numel(k),) if numel(k) else out[k].shape, dtype=out[k].dtype).pin_memory()
                          for k in self.keys},
                 "in_ready": torch.cuda.Event(), "in_free": torch.cuda.Event(), "out_ready": torch.cuda.Event(),
                 "done": torch.cuda.Event()}
            s["in_free"].record(torch.cuda.current_stream(self.dev))
            s["done"].record(torch.cuda.current_stream(self.dev))
            self._slots.append(s)

    @torch.no_grad()
    def submit(self, host_image, im_info=None):
        """host_image: pinned fp32 [1,3,Hp,Wp] (mean-subtracted and padded, like data['data']) with its im_info row (or
        the constructor's), or a pinned raw uint8 [h,w,3] BGR image.  Returns a ticket.  An image the engine cannot
        stage, or one that breaks the combined size rule, raises ValueError before anything is enqueued."""
        from . import operators as ops
        if self._slots is None:
            self._setup(host_image, im_info)
        if (host_image.dtype == torch.uint8) != self.raw:
            raise ValueError("this engine takes %s images" % ("raw uint8" if self.raw else "fp32 blob"))
        g, scale, padded, maps = self._image(host_image, im_info)
        s = self._slots[self._t % self.depth]
        if self.raw and self.sizes is not None:
            H, W = self.max_image_shape
            if host_image.shape[0] > H or host_image.shape[1] > W:
                raise ValueError("image %s larger than max_image_shape %s" % (tuple(host_image.shape[:2]), (H, W)))
        if host_image.numel() > s["in"].numel() or maps[0] * maps[1] > self.map_cap or \
                (self.raw and 3 * padded[0] * padded[1] > s["x"].numel()):
            raise ValueError("image %s does not fit the engine's staging buffers" % (tuple(host_image.shape),))
        n_in = host_image.numel()
        with torch.cuda.stream(self.h2d):
            self.h2d.wait_event(s["in_free"])              # compute has consumed this slot's previous image
            s["in"][:n_in].copy_(host_image.reshape(-1), non_blocking=True)
            s["info"].copy_(torch.from_numpy(g["im_info"]).pin_memory(), non_blocking=True)
            s["in_ready"].record(self.h2d)
        lane = s["lane"]
        cur = self._lane_streams[lane]
        prev_slot = ops.WS_SLOT["i"]
        ops.WS_SLOT["i"] = lane
        try:
            with torch.cuda.stream(cur):
                cur.wait_event(s["in_ready"])
                x = s["in"][:n_in].view(host_image.shape)
                if self.raw:
                    x, _ = ops.prep_image(x, self.pixel_means, scale, self.stride, out=s["x"])
                out, _ = self.model._run_static(x, s["info"], lane=lane)
                out = self._post(dict(out), g)
                s["in_free"].record(cur)
                cur.wait_event(s["done"])                          # this slot's previous results have left the device
                s["shapes"] = {k: tuple(out[k].shape) for k in self.keys}
                for k in self.keys:
                    n = out[k].numel()
                    s["out"][k].view(-1)[:n].copy_(out[k].reshape(-1), non_blocking=True)
                s["out_ready"].record(cur)
        finally:
            ops.WS_SLOT["i"] = prev_slot
        s["im_info"] = g["im_info"]
        with torch.cuda.stream(self.d2h):
            self.d2h.wait_event(s["out_ready"])
            for k in self.keys:
                n = out[k].numel()
                s["host"][k].view(-1)[:n].copy_(s["out"][k].view(-1)[:n], non_blocking=True)
            s["done"].record(self.d2h)
        self._t += 1
        return self._t - 1

    def _post(self, out, g):
        from . import operators as ops
        info = g["im_info"]
        if self.restore_size:
            out["fcn_outputs"], out["panoptic_outputs"] = ops.label_restore(out["fcn_outputs"], info,
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
            boxes = pb[:, 1:] / torch.full((1, 1), float(info[2]), dtype=torch.float32, device=pb.device)
            rle = ops.im_post_rle(boxes, out["mask_probs"], out["cls_inds"], *g["combined_size"], n_dev=n_dev)[:2]
            out["pan_2ch_combined"] = ops.combined_pan_result(out["fcn_outputs"], out["cls_probs"], out["cls_inds"], rle,
                                                              m.num_seg_classes, m.num_classes, *self.combined_thresholds,
                                                              self.stuff_area_limit, n_dev=n_dev, check_errors=False)
        return out

    def result(self, ticket):
        """Blocks until image `ticket` is on the host.  The returned tensors view this slot's pinned buffers at the
        image's own shapes and stay valid until `depth` more images have been submitted; 'im_info' is the row the image
        ran with."""
        assert self._t - self.depth <= ticket < self._t, "result slot already reused (or not yet submitted)"
        s = self._slots[ticket % self.depth]
        s["done"].synchronize()
        h = {k: s["host"][k].view(-1)[:int(np.prod(shape))].view(shape) for k, shape in s["shapes"].items()}
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
        res["im_info"] = torch.from_numpy(s["im_info"].reshape(1, 3).copy())
        return res

    def bytes_per_image(self):
        s = self._slots[0]
        return (s["in"].numel() * s["in"].element_size(), sum(t.numel() * t.element_size() for t in s["host"].values()))
