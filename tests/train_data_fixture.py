"""Synthetic datasets on disk for the training-roidb tests: a VOCdevkit with JPEG images and XML annotations, and a
COCO image set with its instances json.  Seeded; the pixels are smooth noise with a filled rectangle per object, so a
chip and its mirror image differ."""
import json
import os

import numpy as np

VOC_CLASSES = ['aeroplane', 'bicycle', 'bird', 'boat', 'bottle', 'bus', 'car', 'cat', 'chair', 'cow', 'diningtable',
               'dog', 'horse', 'motorbike', 'person', 'pottedplant', 'sheep', 'sofa', 'train', 'tvmonitor']


def _pixels(rng, W, H, boxes):
    im = (rng.rand(H // 8 + 1, W // 8 + 1, 3) * 255).repeat(8, 0).repeat(8, 1)[:H, :W]
    im = im.astype(np.uint8)
    for x1, y1, x2, y2 in boxes:
        im[int(y1):int(y2) + 1, int(x1):int(x2) + 1] = rng.randint(0, 256, 3)
    return im


def _save_jpeg(path, rgb):
    from PIL import Image
    Image.fromarray(rgb).save(path, quality=95)


def _objects(rng, W, H, n, difficult_rate=0.2):
    out = []
    for _ in range(n):
        w, h = int(rng.randint(W // 6, W // 2)), int(rng.randint(H // 6, H // 2))
        x, y = int(rng.randint(1, W - w)), int(rng.randint(1, H - h))
        out.append((VOC_CLASSES[rng.randint(20)], int(rng.rand() < difficult_rate), x, y, x + w, y + h))
    return out


def write_voc(root, sets=(('2007', 'trainval', 3), ('2012', 'trainval', 3), ('2007', 'test', 3)), seed=0,
              size=(320, 240), empty_last=True):
    """VOCdevkit under root with VOC<year>/{Annotations, ImageSets/Main/<set>.txt, JPEGImages}; every image set has its
    own images.  The last image of every trainval set has only difficult objects (empty_last): filter_roidb drops it.
    Returns (devkit path, {'<year>_<set>': [(name, W, H, objects)]})."""
    rng = np.random.RandomState(seed)
    dk = os.path.join(root, 'VOCdevkit')
    listing = {}
    for year, image_set, n in sets:
        vp = os.path.join(dk, 'VOC' + year)
        for sub in ('Annotations', 'ImageSets/Main', 'JPEGImages'):
            os.makedirs(os.path.join(vp, sub), exist_ok=True)
        imgs = []
        for k in range(n):
            name = '%s_%s_%04d' % (year, image_set, k)
            W, H = (size if k % 2 == 0 else size[::-1])
            objs = _objects(rng, W, H, int(rng.randint(1, 4)))
            if empty_last and image_set != 'test' and k == n - 1:
                objs = [o[:1] + (1,) + o[2:] for o in objs]
            elif not any(o[1] == 0 for o in objs):
                objs[0] = objs[0][:1] + (0,) + objs[0][2:]
            xml = ''.join('<object><name>%s</name><difficult>%d</difficult><bndbox><xmin>%d</xmin><ymin>%d</ymin>'
                          '<xmax>%d</xmax><ymax>%d</ymax></bndbox></object>' % o for o in objs)
            with open(os.path.join(vp, 'Annotations', name + '.xml'), 'w') as f:
                f.write('<annotation><size><width>%d</width><height>%d</height><depth>3</depth></size>%s'
                        '</annotation>' % (W, H, xml))
            _save_jpeg(os.path.join(vp, 'JPEGImages', name + '.jpg'),
                       _pixels(rng, W, H, [np.array(o[2:]) - 1 for o in objs]))
            imgs.append((name, W, H, objs))
        with open(os.path.join(vp, 'ImageSets', 'Main', image_set + '.txt'), 'w') as f:
            f.write(''.join(name + '\n' for name, _, _, _ in imgs))
        listing[year + '_' + image_set] = imgs
    return dk, listing


def write_coco(root, image_set='train2014', n=3, seed=1, size=(320, 240)):
    """data_path under root with annotations/instances_<image_set>.json (three categories, one crowd box, one image
    without annotations) and images/<image_set>/COCO_<image_set>_%012d.jpg.  Returns the data path."""
    rng = np.random.RandomState(seed)
    dp = os.path.join(root, 'coco')
    os.makedirs(os.path.join(dp, 'annotations'), exist_ok=True)
    os.makedirs(os.path.join(dp, 'images', image_set), exist_ok=True)
    cats = [dict(id=1, name='person'), dict(id=3, name='car'), dict(id=18, name='dog')]
    images, anns = [], []
    for k in range(n):
        iid = 100 + 7 * k
        W, H = size if k % 2 == 0 else size[::-1]
        images.append(dict(id=iid, width=W, height=H, file_name='COCO_%s_%012d.jpg' % (image_set, iid)))
        boxes = []
        for j, o in enumerate(_objects(rng, W, H, 0 if k == n - 1 else int(rng.randint(1, 4)))):
            bb = [float(o[2]), float(o[3]), float(o[4] - o[2]), float(o[5] - o[3])]
            anns.append(dict(id=len(anns) + 1, image_id=iid, category_id=cats[j % 3]['id'], bbox=bb,
                             area=bb[2] * bb[3], iscrowd=int(k == 0 and j == 0), segmentation=[]))
            boxes.append(o[2:])
        _save_jpeg(os.path.join(dp, 'images', image_set, images[-1]['file_name']), _pixels(rng, W, H, boxes))
    with open(os.path.join(dp, 'annotations', 'instances_%s.json' % image_set), 'w') as f:
        json.dump(dict(images=images, annotations=anns, categories=cats), f)
    return dp
