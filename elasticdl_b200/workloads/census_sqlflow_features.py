"""Feature configuration of the census_model_sqlflow wide & deep models (data of
model_zoo/census_model_sqlflow/wide_and_deep/feature_configs.py:31-268) and their fused GPU transform.

Raw Adult-shaped input with underscore column names: 4 float32 numeric columns and 8 strings.  Each of the three
groups concatenates four features' ids, each offset by the running sum of the bucket counts before it
(feature_configs.py:137-168; no "+1" for a vocabulary: dims 27, 73, 113).  Every cell gives at most one id; an
absent cell is written as -1.  Two id rules (DESIGN.md section 4, Q21-Q25):

  variant="keras"  wide_deep_functional_keras.py, wide_deep_functional_tensor_interface_keras.py,
                   wide_deep_subclass_keras.py: ToSparse drops "" and a numeric 0.0 (absent, no offset);
                   IndexLookup(num_oov_tokens=1) gives an unknown string len(vocabulary) + offset, which is the
                   next feature's id 0 (Q22).
  variant="fc"     wide_deep_functional_fc.py, wide_deep_functional_tensor_interface_fc.py: hash and vocabulary
                   columns drop "" (Q21, recalled); categorical_column_with_vocabulary_list gives an unknown
                   string -1 (Q23, recalled), to which concatenated_categorical_column adds the offset
                   (feature_column.py:157-177): offset - 1, the previous feature's last id, or -1 (pruned, Q24) at
                   offset 0.  Bucketized columns are dense: 0.0 keeps its bucket.
"""
import numpy as np
import torch

from elasticdl_b200.preprocessing.layers import FeatureTransform, encode_strings
from elasticdl_b200.workloads.census_features import synthetic_raw_batch

# feature_configs.py:31-74
WORK_CLASS_VOCABULARY = ["Private", "Self-emp-not-inc", "Self-emp-inc", "Federal-gov", "Local-gov", "State-gov",
                         "Without-pay", "Never-worked"]
MARITAL_STATUS_VOCABULARY = ["Married-civ-spouse", "Divorced", "Never-married", "Separated", "Widowed",
                             "Married-spouse-absent", "Married-AF-spouse"]
RELATION_SHIP_VOCABULARY = ["Wife", "Own-child", "Husband", "Not-in-family", "Other-relative", "Unmarried"]
RACE_VOCABULARY = ["White", "Asian-Pac-Islander", "Amer-Indian-Eskimo", "Other", "Black"]
SEX_VOCABULARY = ["Female", "Male"]
AGE_BOUNDARIES = [0, 20, 40, 60, 80]
CAPITAL_GAIN_BOUNDARIES = [6000, 6500, 7000, 7500, 8000]
CAPITAL_LOSS_BOUNDARIES = [2000, 2500, 3000, 3500, 4000]
HOURS_BOUNDARIES = [10, 20, 30, 40, 50, 60]

# the rows of the numeric float32 [4, B] and strings uint8 [8, B, 32] inputs (feature_configs.py:255-268 names)
NUMERIC_KEYS = ["age", "capital_gain", "capital_loss", "hours_per_week"]
STRING_KEYS = ["workclass", "education", "marital_status", "occupation", "relationship", "race", "sex",
               "native_country"]
STRING_WIDTH = 32

# feature_configs.py:76-134: name -> (op, param)
FEATURES = {
    "education": ("hash", 30),
    "occupation": ("hash", 30),
    "native_country": ("hash", 100),
    "workclass": ("lookup", WORK_CLASS_VOCABULARY),
    "marital_status": ("lookup", MARITAL_STATUS_VOCABULARY),
    "relationship": ("lookup", RELATION_SHIP_VOCABULARY),
    "race": ("lookup", RACE_VOCABULARY),
    "sex": ("lookup", SEX_VOCABULARY),
    "age": ("bucketize", AGE_BOUNDARIES),
    "capital_gain": ("bucketize", CAPITAL_GAIN_BOUNDARIES),
    "capital_loss": ("bucketize", CAPITAL_LOSS_BOUNDARIES),
    "hours_per_week": ("bucketize", HOURS_BOUNDARIES),
}
# feature_configs.py:141-168, in this order
FEATURE_GROUPS = {
    "group1": ["workclass", "hours_per_week", "capital_gain", "capital_loss"],
    "group2": ["education", "marital_status", "relationship", "occupation"],
    "group3": ["age", "sex", "race", "native_country"],
}
VARIANTS = ("keras", "fc")


def num_buckets(name):
    """The bucket count a feature's ids span: hash_bucket_size, len(vocabulary), len(boundaries) + 1."""
    op, param = FEATURES[name]
    return param if op == "hash" else len(param) + (op == "bucketize")


def id_offsets(group):
    """_get_id_offsets_from_dependency_bucket_num (feature_configs.py:137-138)."""
    return [int(v) for v in np.cumsum([0] + [num_buckets(n) for n in FEATURE_GROUPS[group]][:-1])]


GROUP_DIMS = tuple(sum(num_buckets(n) for n in names) for names in FEATURE_GROUPS.values())
assert GROUP_DIMS == (27, 73, 113)
assert [id_offsets(g) for g in FEATURE_GROUPS] == [[0, 8, 15, 21], [0, 30, 37, 43], [0, 6, 8, 13]]


def _check_variant(variant):
    if variant not in VARIANTS:
        raise ValueError("variant must be one of %s, not %r" % (VARIANTS, variant))


def groups(variant):
    """The 12 FeatureTransform group specs of `variant`, group1, group2, group3 in FEATURE_GROUPS order."""
    _check_variant(variant)
    keras = variant == "keras"
    out = []
    for group, names in FEATURE_GROUPS.items():
        for name, off in zip(names, id_offsets(group)):
            op, param = FEATURES[name]
            if op == "lookup":
                spec = {"kind": "lookup", "column": STRING_KEYS.index(name), "vocabulary": param,
                        "num_oov_tokens": 1 if keras else 0, "absent": True}
            elif op == "hash":
                spec = {"kind": "hash", "column": STRING_KEYS.index(name), "num_bins": param, "absent": True}
            else:
                spec = {"kind": "discretize", "column": NUMERIC_KEYS.index(name), "bins": [float(b) for b in param],
                        "absent": keras}
            spec["offset"] = off
            out.append(spec)
    return out


def transform(variant, device=None):
    """The fused feature-id launch of `variant`: ids int32 [12, B] (-1 = absent) from numeric float32 [4, B]
    (NUMERIC_KEYS order) and strings uint8 [8, B, 32] (STRING_KEYS order)."""
    return FeatureTransform(groups(variant), (), torch.int32, device=device)


def synthetic_batch(batch, seed, device, empty_fraction=0.05, zero_fraction=0.05):
    """Seeded Adult-shaped raw rows (census_features.synthetic_raw_batch) with the cells the two id rules treat
    differently made common: about `empty_fraction` of every string column "", about `zero_fraction` of the ages
    and hours 0.0 (capital gains and losses are mostly 0 already).  Returns (numeric float32 [4, B], strings
    uint8 [8, B, 32], raw numeric float32 numpy [4, B], raw strings: 8 lists of str)."""
    _, _, num, raw = synthetic_raw_batch(batch, seed, "cpu")
    rng = np.random.RandomState(seed + 17)
    raw = [["" if rng.rand() < empty_fraction else v for v in col] for col in raw]
    for j in (NUMERIC_KEYS.index("age"), NUMERIC_KEYS.index("hours_per_week")):
        num[j, rng.rand(batch) < zero_fraction] = 0.0
    strings = torch.stack([encode_strings(r, STRING_WIDTH, device="cpu") for r in raw]) if batch else \
        torch.zeros((8, 0, STRING_WIDTH), dtype=torch.uint8)
    return torch.from_numpy(num).to(device), strings.to(device), num, raw
