"""The reference's detect.py loop bodies (detect.py:61-82 images, :118-146 video) written with this package's per-image API --
val_aug, net(img[None]), nms, after_nms(..., img_name), draw_img.  Batched detection must hand cv2.imwrite and
VideoWriter.write exactly what these loops hand them."""
import cv2
import torch

from yolact_minimal_b200.utils.augmentations import val_aug
from yolact_minimal_b200.utils.output_utils import after_nms, draw_img, nms


def _one(net, cfg, img_origin, img_name, fps=None):
    dev = next(net.parameters()).device
    img_h, img_w = img_origin.shape[0:2]
    with torch.no_grad():
        class_p, box_p, coef_p, proto_p = net(val_aug(img_origin, cfg.img_size, dev)[None])
    ids_p, class_p, box_p, coef_p, proto_p = nms(class_p, box_p, coef_p, proto_p, net.anchors, cfg)
    ids_p, class_p, boxes_p, masks_p = after_nms(ids_p, class_p, box_p, coef_p, proto_p, img_h, img_w, cfg, img_name=img_name)
    return draw_img(ids_p, class_p, boxes_p, masks_p, img_origin, cfg, img_name=img_name, fps=fps)


def per_image_detect(net, cfg, paths):
    """paths: the sorted *.jpg files, read with cv2.imread as the reference's COCODetection(mode='detect') does."""
    for path in paths:
        name = path.split('/')[-1]
        cv2.imwrite(f'results/images/{name}', _one(net, cfg, cv2.imread(path), name))


def per_frame_detect(net, cfg, video, writer):
    vid = cv2.VideoCapture(video)
    for _ in range(round(vid.get(cv2.CAP_PROP_FRAME_COUNT))):
        frame_origin = vid.read()[1]
        writer.write(_one(net, cfg, frame_origin, None, fps=0))
    vid.release()
