"""Golden of the COCO result format: COCOEvaluator.convert_to_coco_format (unicorn/evaluators/coco_evaluator.py:128-158) of the
UNMODIFIED reference on fixed postprocess rows of two images of different sizes (build container only).

    python tests/golden/make_golden_coco.py      (writes tests/golden/coco_detections.json)"""
import json
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle"))
import ref_import  # noqa: E402

# the 80 COCO category ids in the order of the contiguous class index (COCODataset.class_ids = sorted(coco.getCatIds()))
CLASS_IDS = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 27, 28, 31, 32, 33, 34, 35, 36, 37, 38,
             39, 40, 41, 42, 43, 44, 46, 47, 48, 49, 50, 51, 52, 53, 54, 55, 56, 57, 58, 59, 60, 61, 62, 63, 64, 65, 67, 70, 72, 73, 74, 75,
             76, 77, 78, 79, 80, 81, 82, 84, 85, 86, 87, 88, 89, 90]
IMG_SIZE = (800, 1280)


def main():
    ref_import.install()
    # the module file itself: the evaluators package also imports the BDD / MOT evaluators and their third-party dependencies
    import importlib.util
    spec = importlib.util.spec_from_file_location("coco_evaluator", os.path.join(ref_import.REF_ROOT, "unicorn", "evaluators", "coco_evaluator.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    COCOEvaluator = mod.COCOEvaluator
    g = torch.Generator().manual_seed(7)
    images = [(480, 640, 139), (427, 612, 785)]  # (h, w, image id)
    rows = []
    for _ in images:
        n = 6
        xy = torch.rand(n, 2, generator=g) * 700
        wh = torch.rand(n, 2, generator=g) * 300 + 1
        r = torch.cat([xy, xy + wh, torch.rand(n, 2, generator=g), torch.randint(0, 80, (n, 1), generator=g).float()], 1)
        rows.append(r)
    ev = object.__new__(COCOEvaluator)
    ev.img_size = IMG_SIZE
    ev.dataloader = types.SimpleNamespace(dataset=types.SimpleNamespace(class_ids=CLASS_IDS))
    info = ([h for h, _, _ in images], [w for _, w, _ in images])
    data = ev.convert_to_coco_format([r.clone() for r in rows], info, [i for _, _, i in images])
    with open(os.path.join(HERE, "coco_detections.json"), "w") as f:
        json.dump(dict(img_size=IMG_SIZE, images=images, class_ids=CLASS_IDS, rows=[r.tolist() for r in rows], coco=data), f)
    print(len(data), "detections")


if __name__ == "__main__":
    main()
