"""COCO category tables the EfficientDet path needs (reference: class_ids.py:526-549 `coco_id_mapping`, efficientdet_wrapper.py:476-508
`coco_id_mapping_reverse`; obj_detect_tracking.py:636-647 maps the 1..90 category ids back to the 1..80 class ids).
The 80 COCO "thing" categories keep their sparse 1..90 ids; index in COCO_NAMES + 1 is the dense 1..80 class id."""

COCO_NAMES = (
    "person bicycle car motorcycle airplane bus train truck boat|traffic light|fire hydrant|stop sign|parking meter|"
    "bench bird cat dog horse sheep cow elephant bear zebra giraffe backpack umbrella handbag tie suitcase frisbee skis "
    "snowboard|sports ball|kite|baseball bat|baseball glove|skateboard surfboard|tennis racket|bottle|wine glass|"
    "cup fork knife spoon bowl banana apple sandwich orange broccoli carrot|hot dog|pizza donut cake chair couch|"
    "potted plant|bed|dining table|toilet tv laptop mouse remote keyboard|cell phone|microwave oven toaster sink "
    "refrigerator book clock vase scissors|teddy bear|hair drier|toothbrush")


def _split(spec):
    out = []
    for chunk in spec.split("|"):
        chunk = chunk.strip()
        # multi-word names are their own '|' chunk; the rest are space separated single words
        if " " in chunk and chunk in ("traffic light", "fire hydrant", "stop sign", "parking meter", "sports ball",
                                      "baseball bat", "baseball glove", "tennis racket", "wine glass", "hot dog",
                                      "potted plant", "dining table", "cell phone", "teddy bear", "hair drier"):
            out.append(chunk)
        else:
            out.extend(chunk.split())
    return out


_MISSING = (12, 26, 29, 30, 45, 66, 68, 69, 71, 83)                   # ids COCO never assigned
coco_obj_classes = ["BG"] + _split(COCO_NAMES)                        # dense ids 0..80
coco_ids = [i for i in range(1, 91) if i not in _MISSING]             # sparse ids of the 80 categories
coco_id_mapping = dict(zip(coco_ids, coco_obj_classes[1:]))          # 1..90 -> name
coco_id_mapping_reverse = {v: k for k, v in coco_id_mapping.items()}  # name -> 1..90
coco_obj_class_to_id = {n: i for i, n in enumerate(coco_obj_classes)}
coco_obj_id_to_class = {i: n for n, i in coco_obj_class_to_id.items()}
assert len(coco_obj_classes) == 81 and len(coco_ids) == 80

# class_ids.py:551-558: the COCO classes the ActEV drivers track and the ActEV object each stands for.  Its keys, in this
# order, are the default partial_classes of --use_partial_classes (obj_detect_tracking.py:237-239).
coco_obj_to_actev_obj = {
    "person": "Person",
    "car": "Vehicle",
    "bus": "Vehicle",
    "truck": "Vehicle",
    "bicycle": "Bike",
}


# class_ids.py:99-117: the ActEV merge-prop model's 17 classes (main.py --merge_prop), the table the small-object head
# resolves its class names through (main.py:506-521)
MERGE_PROP_NAMES = (
    "BG Vehicle Person Parking_Meter Tree Other Trees Construction_Barrier Door Dumpster Push_Pulled_Object "
    "Construction_Vehicle Prop Bike Animal Articulated_Infrastructure Prop_plus_Push_Pulled_Object")
targetClass2id_mergeProp = {n: i for i, n in enumerate(MERGE_PROP_NAMES.split())}
assert len(targetClass2id_mergeProp) == 17

# main.py:506-507: the default small_objects of --use_small_object_head
SMALL_OBJECTS = ("Prop", "Push_Pulled_Object", "Prop_plus_Push_Pulled_Object", "Bike")


def effdet_labels_to_coco80(labels):
    """obj_detect_tracking.py:644-647: EfficientDet's 1..90 category ids -> the detector's dense 1..80 class ids."""
    return [coco_obj_class_to_id[coco_id_mapping[int(l)]] for l in labels]
