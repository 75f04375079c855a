"""Feature configuration of the census wide & deep model zoo entry (data of
model_zoo/census_wide_deep_model/feature_config.py:21-122, composed as in wide_deep_functional_api.py:120-161 and
feature_info_util.py:25-40) and its fused GPU transform.

Raw Adult-dataset-shaped input: 4 numeric columns (tf.float32 features) and 8 categorical strings.  Each group
concatenates its features' ids, each offset by get_id_boundaries (the running sum of get_max_id: len(vocabulary) + 1
for LOOKUP and BUCKETIZE, the bucket count for HASH).  LOOKUP is CategoryLookup (keras_process_layer.py:55-65):
index_table_from_tensor with one OOV bucket, which is IndexLookup(vocabulary, num_oov_tokens=1)."""
import numpy as np
import torch

from elasticdl_b200.preprocessing.layers import FeatureTransform, encode_strings

# feature_config.py:21-59
WORK_CLASS_VOCABULARY = ["Private", "Self-emp-not-inc", "Self-emp-inc", "Federal-gov", "Local-gov", "State-gov",
                         "Without-pay", "Never-worked"]
MARITAL_STATUS_VOCABULARY = ["Married-civ-spouse", "Divorced", "Never-married", "Separated", "Widowed",
                             "Married-spouse-absent", "Married-AF-spouse"]
RELATION_SHIP_VOCABULARY = ["Wife", "Own-child", "Husband", "Not-in-family", "Other-relative", "Unmarried"]
RACE_VOCABULARY = ["White", "Asian-Pac-Islander", "Amer-Indian-Eskimo", "Other", "Black"]
SEX_VOCABULARY = ["Female", "Male"]
# feature_config.py:61-64
AGE_BOUNDARIES = [0, 20, 40, 60, 80]
CAPITAL_GAIN_BOUNDARIES = [6000, 6500, 7000, 7500, 8000]
CAPITAL_LOSS_BOUNDARIES = [2000, 2500, 3000, 3500, 4000]
HOURS_BOUNDARIES = [10, 20, 30, 40, 50, 60]

# feature_config.py:106-121: the input column order
CATEGORICAL_FEATURE_KEYS = ["workclass", "education", "marital-status", "occupation", "relationship", "race", "sex",
                            "native-country"]
NUMERIC_FEATURE_KEYS = ["age", "capital-gain", "capital-loss", "hours-per-week"]

# feature_config.py:66-93: name -> (op, param)
FEATURES = {
    "education": ("hash", 30),
    "occupation": ("hash", 30),
    "native-country": ("hash", 100),
    "workclass": ("lookup", WORK_CLASS_VOCABULARY),
    "marital-status": ("lookup", MARITAL_STATUS_VOCABULARY),
    "relationship": ("lookup", RELATION_SHIP_VOCABULARY),
    "race": ("lookup", RACE_VOCABULARY),
    "sex": ("lookup", SEX_VOCABULARY),
    "age": ("bucketize", AGE_BOUNDARIES),
    "capital-gain": ("bucketize", CAPITAL_GAIN_BOUNDARIES),
    "capital-loss": ("bucketize", CAPITAL_LOSS_BOUNDARIES),
    "hours-per-week": ("bucketize", HOURS_BOUNDARIES),
}
# feature_config.py:95-99
FEATURE_GROUPS = {
    "group1": ["workclass", "hours-per-week", "capital-gain", "capital-loss"],
    "group2": ["education", "marital-status", "relationship", "occupation"],
    "group3": ["age", "sex", "race", "native-country"],
}
STRING_WIDTH = 32


def max_id(name):
    """feature_info_util.py:32-40 (get_max_id)."""
    op, param = FEATURES[name]
    return param if op == "hash" else len(param) + 1


def id_offsets(group):
    """feature_info_util.py:25-29 (get_id_boundaries) without its last entry, the group's dimension."""
    out = [0]
    for name in FEATURE_GROUPS[group]:
        out.append(out[-1] + max_id(name))
    return out[:-1]


ID_GROUP_DIMS = {g: id_offsets(g)[-1] + max_id(FEATURE_GROUPS[g][-1]) for g in FEATURE_GROUPS}
assert ID_GROUP_DIMS == {"group1": 28, "group2": 75, "group3": 115}  # wide_deep_functional_api.py:156-161
assert [id_offsets(g) for g in FEATURE_GROUPS] == [[0, 9, 16, 22], [0, 30, 38, 45], [0, 6, 9, 15]]


def census_groups():
    """The 12 FeatureTransform group specs, group1, group2, group3 in FEATURE_GROUPS order."""
    groups = []
    for group, names in FEATURE_GROUPS.items():
        for name, off in zip(names, id_offsets(group)):
            op, param = FEATURES[name]
            if op == "lookup":
                spec = {"kind": "lookup", "column": CATEGORICAL_FEATURE_KEYS.index(name), "vocabulary": param,
                        "num_oov_tokens": 1}
            elif op == "hash":
                spec = {"kind": "hash", "column": CATEGORICAL_FEATURE_KEYS.index(name), "num_bins": param}
            else:
                spec = {"kind": "discretize", "column": NUMERIC_FEATURE_KEYS.index(name), "bins": [float(b) for b in param]}
            spec["offset"] = off
            groups.append(spec)
    return groups


def census_transform(ids_dtype=torch.int64, device=None):
    """transform(inputs, FEATURE_GROUPS) in one launch: ids [12, B] from numeric float32 [4, B]
    (NUMERIC_FEATURE_KEYS order) and strings uint8 [8, B, 32] (CATEGORICAL_FEATURE_KEYS order)."""
    return FeatureTransform(census_groups(), (), ids_dtype, device=device)


def synthetic_raw_batch(batch, seed, device):
    """Seeded Adult-shaped raw values.  Lookup columns draw vocabulary terms, about 5 % "?" (Adult's missing marker)
    and some unseen strings; hashed columns draw free strings.  Ages 17-90, capital gains and losses mostly 0,
    hours 1-99, and every boundary value exactly (where the batch has room), so the left-closed bins are exercised.
    Returns (numeric float32 [4, B], strings uint8 [8, B, 32], raw numeric numpy [4, B], raw string lists)."""
    rng = np.random.RandomState(seed)
    age = rng.randint(17, 91, batch).astype(np.float32)
    gain = np.where(rng.rand(batch) < 0.9, 0, rng.randint(1, 20000, batch)).astype(np.float32)
    loss = np.where(rng.rand(batch) < 0.95, 0, rng.randint(1, 5000, batch)).astype(np.float32)
    hours = rng.randint(1, 100, batch).astype(np.float32)
    num = np.stack([age, gain, loss, hours])
    for j, name in enumerate(NUMERIC_FEATURE_KEYS):
        b = np.asarray(FEATURES[name][1], dtype=np.float32)
        k = min(len(b), batch)
        num[j, rng.choice(batch, k, replace=False)] = b[:k]
    raw = []
    for name in CATEGORICAL_FEATURE_KEYS:
        op, param = FEATURES[name]
        if op == "lookup":
            pool = np.array(param + ["?", "Unseen-" + name, "private", ""], dtype=object)
            p = np.full(len(pool), 0.88 / len(param))
            p[len(param):] = [0.05, 0.03, 0.02, 0.02]
            vals = pool[rng.choice(len(pool), batch, p=p / p.sum())]
        else:
            n = rng.randint(1, STRING_WIDTH + 1, batch)
            vals = np.array(["%s-%x" % (name, v) for v in rng.randint(0, 1 << 30, batch)], dtype=object)
            vals = np.array([v[:k] for v, k in zip(vals, n)], dtype=object)
            vals[rng.rand(batch) < 0.05] = "?"
        raw.append([str(v) for v in vals])
    strings = torch.stack([encode_strings(r, STRING_WIDTH, device="cpu") for r in raw]) if batch else \
        torch.zeros((8, 0, STRING_WIDTH), dtype=torch.uint8)
    return torch.from_numpy(num).to(device), strings.to(device), num, raw
