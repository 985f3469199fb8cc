"""Record what the plugin-surface test compares against, from the UNMODIFIED reference staged under oracle/_ref:
the LightGlue state_dict layout (names, shapes) and confidence thresholds, and the homography ground-truth component's
required keys and default configuration -> tests/golden/reference_plugin_surface.json.

    python -m oracle.make_surface_golden
"""
import json
import os

from oracle import stage_reference

OUT = os.path.join(stage_reference.ROOT, "tests", "golden", "reference_plugin_surface.json")


def main():
    get_model = stage_reference.import_reference()
    assert get_model is not None, "stage the reference first (oracle/stage_reference.py)"
    ref = get_model("matchers.lightglue")({"n_layers": 2})
    gt = get_model("matchers.homography_matcher")
    out = {
        "lightglue_n_layers2": {
            "keys": list(ref.state_dict().keys()),
            "shapes": [list(v.shape) for v in ref.state_dict().values()],
            "confidence_thresholds": ref.confidence_thresholds.tolist(),
        },
        "homography_matcher": {
            "required_data_keys": sorted(gt({}).required_data_keys),
            "default_conf": json.loads(json.dumps(dict(gt.default_conf))),
        },
    }
    with open(OUT, "w") as f:
        json.dump(out, f)
        f.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
