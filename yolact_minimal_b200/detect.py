"""Detection in batches on the GPU: the reference's detect.py with the same arguments and outputs (results/images/{name},
lincomb_{name}, the cutout images, results/videos/{name}), fed `--det_bs` images or video frames at a time:

    one H2D copy -> val_aug_batch -> net(images) -> detect_batched -> visible_count -> after_nms_batched
      -> blend_masks_batched (unless hide_mask) -> lincomb_batched (save_lincomb) -> async D2H copies        (per batch, no host sync)
    draw_labels (cv2 boxes, labels, fps) -> cv2.imwrite / VideoWriter.write                                  (host, one batch behind)

The host waits for batch i only after batch i+1 is queued, so the cv2 pass of one batch runs under the device work of the next.
With --jpeg_gpu the image files are encoded on the device (yb_jpeg_encode_batch, the bytes cv2.imwrite writes): the drawn images
of a batch go into one page-locked buffer, one H2D copy, one encode and one D2H copy on a stream of their own, and the files are
written one batch later; lincomb_{name} and the cutout images are encoded where they are, on the device.
With --decode_gpu the loader's workers read the files' bytes instead of decoding them, and a batch's JPEG files are decoded on the
device (yb_jpeg_decode_batch, the pixels cv2.imread returns) in place of the H2D copy of its pixels; files it refuses are read by
cv2.imread in the workers as before.  A file with corrupt entropy-coded data raises once its batch has run.
Every written image equals the reference's per-image loop (val_aug, net, nms, after_nms, draw_img) on this package bit for bit:
the forward is batch-invariant at a fixed max_batch, detect_batched treats images independently, visual_thre keeps a prefix of
each image's score-sorted detections, after_nms_batched equals after_nms per image and bit-packed masks draw as float masks do.

    python -m yolact_minimal_b200.detect --weight weights/best_30.5_res101_coco_392000.pth --image images --det_bs 16
"""
import argparse
import re
import time

import torch

from . import _lib
from .utils.augmentations import val_aug_batch
from .utils.coco import DetectImages, PackedDetectBatch, detect_collate
from .utils.common_utils import ProgressBar
from .utils.output_utils import (after_nms_batched, blend_masks_batched, cutout_masks, cutout_masks_device, detect_batched, draw_labels,
                                 imencode_batched, lincomb_batched, visible_count)


class _HostBuffers:
    """Page-locked buffers the D2H copies of one batch land in; detect keeps two and alternates, so a batch's results stay put
    while the next batch's copies are queued."""

    def __init__(self):
        self._bufs = {}

    def take(self, key, t):
        buf = self._bufs.get(key)
        if buf is None or buf.numel() < t.numel() or buf.dtype != t.dtype:
            buf = self._bufs[key] = torch.empty(t.numel(), dtype=t.dtype, pin_memory=True)
        buf = buf[:t.numel()]
        buf.copy_(t.reshape(-1), non_blocking=True)
        return buf.view(t.shape)


class JpegWriter:
    """Writes JPEG files encoded on the device, byte for byte what cv2.imwrite(path, img) writes.  A batch's files are collected
    with put_host (host images: packed into one page-locked buffer) and put_device (images already on the device), then flush(after)
    queues their encodes on the writer's own stream behind the event `after`, with one D2H copy per encode, and writes the previous
    batch's files.  close() writes the last batch's."""

    def __init__(self, quality=95):
        self.quality = quality
        self.stream = torch.cuda.Stream()
        self._host, self._device, self._pending = [], [], None

    def put_host(self, path, img):
        self._host.append((path, img))

    def put_device(self, paths, buffer, items, keep=None):
        """paths[i] receives image items[i] (yb_val_aug_item layout) of the CUDA uint8 `buffer`; `keep` (e.g. the tensors a kernel
        queued on the writer's stream reads) is held until the files are written."""
        self._device.append((list(paths), buffer, items, keep))

    def _encode(self, paths, buffer, items, keep):
        data, off, lengths = imencode_batched(buffer, items, self.quality)
        data_h = torch.empty(data.numel(), dtype=torch.uint8, pin_memory=True)
        len_h = torch.empty(lengths.numel(), dtype=torch.int64, pin_memory=True)
        data_h.copy_(data, non_blocking=True)
        len_h.copy_(lengths, non_blocking=True)
        return paths, off, data_h, len_h, (data, buffer, keep)

    def flush(self, after=None):
        import numpy as np
        from .utils.augmentations import VAL_ITEM_DTYPE
        jobs = []
        with torch.cuda.stream(self.stream):
            if after is not None:
                self.stream.wait_event(after)
            if self._host:
                items = np.zeros(len(self._host), VAL_ITEM_DTYPE)
                buf = torch.empty(sum(img.nbytes for _, img in self._host), dtype=torch.uint8, pin_memory=True)
                flat, o = buf.numpy(), 0
                for i, (_, img) in enumerate(self._host):
                    flat[o:o + img.nbytes] = np.ascontiguousarray(img).reshape(-1)
                    items[i] = (o, img.shape[0], img.shape[1])
                    o += img.nbytes
                src = buf.to(torch.cuda.current_device(), non_blocking=True)
                jobs.append(self._encode([p for p, _ in self._host], src, items, buf))
            for paths, buffer, items, keep in self._device:
                jobs.append(self._encode(paths, buffer, items, keep))
            done = torch.cuda.Event()
            done.record()
        self._host, self._device = [], []
        self._write()
        self._pending = (jobs, done)

    def _write(self):
        if self._pending is None:
            return
        jobs, done = self._pending
        done.synchronize()
        for paths, off, data_h, len_h, _ in jobs:
            data, lens = data_h.numpy(), len_h.numpy()
            for i, path in enumerate(paths):
                with open(path, 'wb') as f:
                    f.write(data[off[i]:off[i] + lens[i]].tobytes())
        self._pending = None

    def close(self):
        self.flush()
        self._write()


class _Pending:
    """A queued batch: what its host pass needs once `done` has completed."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def enqueue(net, cfg, packed, host):
    """Queues one batch's device work and the copies of its results into `host` (a _HostBuffers); never waits for the device."""
    dev = next(net.parameters()).device
    decoded = packed.buffer is None
    src, status = packed.to_device(dev)
    with torch.no_grad():
        images = val_aug_batch(src, packed.items, cfg.img_size, dev)
        class_p, box_p, coef_p, proto_p = net(images)
    det = detect_batched(class_p, box_p, coef_p, net.anchors, cfg)
    det = dict(det, count=visible_count(det, cfg.visual_thre))
    boxes_px, masks = after_nms_batched(det, proto_p, packed.sizes, crop=not cfg.no_crop)
    out = {'count': det['count'], 'cls': det['cls'], 'score': det['score'], 'boxes': boxes_px}
    if not cfg.hide_mask:
        out['frames'] = blend_masks_batched(src, packed.items, det, masks, cfg.num_classes)
    lincomb = None
    if cfg.save_lincomb:
        lincomb = lincomb_batched(proto_p, det)
        if not getattr(cfg, 'jpeg_gpu', False):
            out['lincomb'] = lincomb
            lincomb = None
    if decoded:
        out['pixels'] = src                               # the host pass draws on (and emits) the decoded pixels
        if status is not None:
            out['status'] = status
    res = {k: host.take(k, v) for k, v in out.items()}
    if decoded:
        packed.buffer = res['pixels']
    done = torch.cuda.Event()
    done.record()
    return _Pending(packed=packed, src=src, det=det, masks=masks, res=res, done=done, lincomb=lincomb)


def _put_cutouts(writer, p, b, n, boxes_np, cfg):
    """The cutout images of image b, cut and encoded on the writer's stream without leaving the device."""
    import numpy as np
    from .utils.augmentations import VAL_ITEM_DTYPE
    h, w = p.packed.sizes[b]
    off, name = int(p.packed.items[b]['img_off']), p.packed.names[b]
    with torch.cuda.stream(writer.stream):
        writer.stream.wait_event(p.done)
        src_b = p.src[off:off + h * w * 3].view(h, w, 3)
        total, crops, coff, shapes = cutout_masks_device(src_b, p.det['cls'][b, :n], boxes_np, p.masks[b][:n], cfg.num_classes)
    writer.put_device([f'results/images/{name}_total_obj.jpg'], total.view(-1), np.array([(0, h, w)], VAL_ITEM_DTYPE), keep=p)
    if shapes:
        items = np.array([(coff[i], ch, cw) for i, (ch, cw) in enumerate(shapes)], VAL_ITEM_DTYPE)
        writer.put_device([f'results/images/{name}_{i}.jpg' for i in range(len(shapes))], crops, items)


def finish(p, cfg, emit, fps=None, writer=None):
    """Waits for a queued batch and runs the host pass of draw_img on each image: lincomb_{name} (save_lincomb), the cutout images,
    then the boxes / labels / fps; emit(name, image) receives each drawn image.  With a JpegWriter the lincomb and cutout images
    are encoded on the device and the writer is flushed after the batch."""
    import cv2
    import numpy as np
    p.done.synchronize()
    r, packed = p.res, p.packed
    if 'status' in r:
        bad = [packed.names[int(packed.mixed.encoded[k])] for k in np.flatnonzero(r['status'].numpy())]
        if bad:
            raise RuntimeError(f'corrupt JPEG data in {", ".join(str(b) for b in bad)}')
    count = r['count'].numpy()
    for b, (h, w) in enumerate(packed.sizes):
        n, name = int(count[b]), packed.names[b]
        if n <= 0:                                        # after_nms returned None: draw_img gives back img_origin
            emit(name, packed.image(b))
            continue
        if cfg.save_lincomb and writer is not None:
            _, H, W, _ = p.lincomb.shape
            writer.put_device([f'results/images/lincomb_{name}'], p.lincomb.view(-1),
                              np.array([(b * H * W * 3, H, W)], np.dtype(_lib.ValAugItem)))
        elif cfg.save_lincomb:
            cv2.imwrite(f'results/images/lincomb_{name}', r['lincomb'][b].numpy())
        ids_np, scores_np, boxes_np = r['cls'][b, :n].numpy(), r['score'][b, :n].numpy(), r['boxes'][b, :n].numpy()
        if cfg.hide_mask:
            img = packed.image(b)                         # drawn in place, as the reference draws into img_origin
        else:
            off = int(packed.items[b]['img_off'])
            if cfg.cutout and writer is not None:
                _put_cutouts(writer, p, b, n, boxes_np, cfg)
            elif cfg.cutout:
                src_b = p.src[off:off + h * w * 3].view(h, w, 3)
                total, crops = cutout_masks(src_b, p.det['cls'][b, :n], boxes_np, p.masks[b][:n], cfg.num_classes)
                cv2.imwrite(f'results/images/{name}_total_obj.jpg', total)
                for i, crop in enumerate(crops):
                    cv2.imwrite(f'results/images/{name}_{i}.jpg', crop)
            img = r['frames'][off:off + h * w * 3].numpy().reshape(h, w, 3)
        emit(name, draw_labels(img, ids_np, scores_np, boxes_np, cfg, fps))
    if writer is not None:
        writer.flush(p.done)


def run(net, cfg, batches, emit, progress=None, writer=None):
    """Detects every batch of `batches` (PackedDetectBatch) with one batch in flight while the host draws the previous one.
    progress(done_images, images_per_second) is called after each batch; the rate is also the fps the real_time view shows."""
    hosts = (_HostBuffers(), _HostBuffers())
    pending, done, start, fps = None, 0, time.perf_counter(), 0.0
    for i, packed in enumerate(batches):
        cur = enqueue(net, cfg, packed, hosts[i % 2])
        if pending is not None:
            finish(pending, cfg, emit, fps, writer)
            done += len(pending.packed)
            fps = done / (time.perf_counter() - start)
            if progress:
                progress(done, fps)
        pending = cur
    if pending is not None:
        finish(pending, cfg, emit, fps, writer)
        done += len(pending.packed)
        if progress:
            progress(done, done / (time.perf_counter() - start))


def detect_images(net, cfg, det_bs, num_workers=2):
    """The reference's image loop (detect.py:52-99): every cfg.image/*.jpg, drawn to results/images/{name}."""
    import cv2
    from torch.utils.data import DataLoader
    dataset = DetectImages(cfg, decode_gpu=getattr(cfg, 'decode_gpu', False))
    assert len(dataset) > 0, 'No .jpg images found.'
    loader = DataLoader(dataset, det_bs, num_workers=num_workers, shuffle=False, pin_memory=True, collate_fn=detect_collate)
    bar = ProgressBar(40, len(dataset))

    def progress(done, fps):
        print(f'\rTesting: {bar.get_bar(done)} {done}/{len(dataset)}, total fps: {fps:.2f}', end='')

    if getattr(cfg, 'jpeg_gpu', False):
        writer = JpegWriter()
        run(net, cfg, loader, lambda name, img: writer.put_host(f'results/images/{name}', img), progress, writer)
        writer.close()
    else:
        run(net, cfg, loader, lambda name, img: cv2.imwrite(f'results/images/{name}', img), progress)
    print('\nFinished, saved in: results/images.')


def _video_batches(vid, num_frames, det_bs):
    frames = []
    for _ in range(num_frames):
        ok, frame = vid.read()
        if not ok:
            break
        frames.append(frame)
        if len(frames) == det_bs:
            yield PackedDetectBatch(frames, [None] * len(frames)).pin_memory()     # the reference names no frame
            frames = []
    if frames:
        yield PackedDetectBatch(frames, [None] * len(frames)).pin_memory()


def detect_video(net, cfg, det_bs):
    """The reference's video loop (detect.py:101-167): frames to results/videos/{name} (mp4v), or to a window with real_time."""
    import cv2
    vid = cv2.VideoCapture(cfg.video)
    target_fps = round(vid.get(cv2.CAP_PROP_FPS))
    frame_width = round(vid.get(cv2.CAP_PROP_FRAME_WIDTH))
    frame_height = round(vid.get(cv2.CAP_PROP_FRAME_HEIGHT))
    num_frames = round(vid.get(cv2.CAP_PROP_FRAME_COUNT))
    name = cfg.video.split('/')[-1]
    video_writer = cv2.VideoWriter(f'results/videos/{name}', cv2.VideoWriter_fourcc(*"mp4v"), target_fps, (frame_width, frame_height))
    bar = ProgressBar(40, max(num_frames, 1))

    def emit(_, frame):
        if cfg.real_time:
            cv2.imshow('Detection', frame)
            cv2.waitKey(1)
        else:
            video_writer.write(frame)

    def progress(done, fps):
        print(f'\rDetecting: {bar.get_bar(done)} {done}/{num_frames}, total fps: {fps:.2f}', end='')

    run(net, cfg, _video_batches(vid, num_frames, det_bs), emit, progress)
    if not cfg.real_time:
        print(f'\n\nFinished, saved in: results/videos/{name}')
    vid.release()
    video_writer.release()


def main(argv=None):
    from .config import get_config
    from .modules.yolact import Yolact
    parser = argparse.ArgumentParser(description='YOLACT Detection.')
    parser.add_argument('--weight', default='weights/best_30.5_res101_coco_392000.pth', type=str)
    parser.add_argument('--image', default=None, type=str, help='The folder of images for detecting.')
    parser.add_argument('--video', default=None, type=str, help='The path of the video to evaluate.')
    parser.add_argument('--img_size', type=int, default=544, help='The image size for validation.')
    parser.add_argument('--traditional_nms', default=False, action='store_true', help='Whether to use traditional nms.')
    parser.add_argument('--hide_mask', default=False, action='store_true', help='Hide masks in results.')
    parser.add_argument('--hide_bbox', default=False, action='store_true', help='Hide boxes in results.')
    parser.add_argument('--hide_score', default=False, action='store_true', help='Hide scores in results.')
    parser.add_argument('--cutout', default=False, action='store_true', help='Cut out each object and save.')
    parser.add_argument('--save_lincomb', default=False, action='store_true', help='Show the generating process of masks.')
    parser.add_argument('--no_crop', default=False, action='store_true',
                        help='Do not crop the output masks with the predicted bounding box.')
    parser.add_argument('--real_time', default=False, action='store_true', help='Show the detection results real-timely.')
    parser.add_argument('--visual_thre', default=0.3, type=float,
                        help='Detections with a score under this threshold will be removed.')
    parser.add_argument('--det_bs', default=1, type=int, help='Images (or video frames) per batch on the GPU.')
    parser.add_argument('--jpeg_gpu', default=False, action='store_true',
                        help='Encode the image files on the GPU (the same bytes cv2.imwrite writes).')
    parser.add_argument('--decode_gpu', default=False, action='store_true',
                        help='Decode the input JPEG files on the GPU (the same pixels cv2.imread returns).')
    args = parser.parse_args(argv)
    if args.det_bs < 1:
        parser.error(f'--det_bs must be >= 1, got {args.det_bs}')
    prefix = re.findall(r'best_\d+\.\d+_', args.weight)[0]
    suffix = re.findall(r'_\d+\.pth', args.weight)[0]
    args.cfg = args.weight.split(prefix)[-1].split(suffix)[0]
    cfg = get_config(args, mode='detect')
    cfg.max_batch = args.det_bs                      # the forward is batch-invariant at a fixed max_batch

    net = Yolact(cfg)
    net.load_weights(cfg.weight, cfg.cuda)
    net.eval()
    net = net.cuda()
    if cfg.image is not None:
        detect_images(net, cfg, args.det_bs)
    elif cfg.video is not None:
        detect_video(net, cfg, args.det_bs)


if __name__ == '__main__':
    main()
