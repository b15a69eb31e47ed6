"""The reference's per-image evaluation loop (eval.py:42-69,106) written with this package's per-image API -- val_aug,
net(img[None]), nms, after_nms with float masks, prep_metrics, calc_map -- over a COCOValDetection-style dataset.  The batched
evaluate() must return exactly its (table, box_row, mask_row)."""
import torch

from yolact_minimal_b200.eval import iou_thres
from yolact_minimal_b200.utils.augmentations import val_aug
from yolact_minimal_b200.utils.common_utils import APDataObject, calc_map, prep_metrics
from yolact_minimal_b200.utils.mask_utils import unpack_masks
from yolact_minimal_b200.utils.output_utils import after_nms, nms


def per_image_evaluate(net, cfg, samples, step=None):
    """samples: iterable of COCOValDetection items (img_u8, gt [n,5], packed gt masks, (h, w), id)."""
    dev = next(net.parameters()).device
    ap_data = {'box': [[APDataObject() for _ in cfg.class_names] for _ in iou_thres],
               'mask': [[APDataObject() for _ in cfg.class_names] for _ in iou_thres]}
    for img, gt, gt_bits, (img_h, img_w), _ in samples:
        with torch.no_grad():
            class_p, box_p, coef_p, proto_p = net(val_aug(img, cfg.img_size, dev)[None])
        ids_p, class_p, box_p, coef_p, proto_p = nms(class_p, box_p, coef_p, proto_p, net.anchors, cfg)
        ids_p, class_p, boxes_p, masks_p = after_nms(ids_p, class_p, box_p, coef_p, proto_p, img_h, img_w)
        if ids_p is None:
            continue
        ids_p = list(ids_p.cpu().numpy().astype(int))
        class_p = list(class_p.cpu().numpy().astype(float))
        gt_masks = unpack_masks(torch.from_numpy(gt_bits).to(dev), img_w).float()
        prep_metrics(ap_data, ids_p, class_p, boxes_p, masks_p, torch.from_numpy(gt).to(dev), gt_masks, img_h, img_w, iou_thres)
    return calc_map(ap_data, iou_thres, len(cfg.class_names), step=step)
