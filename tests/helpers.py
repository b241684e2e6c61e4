"""Shared test helpers (CPU + GPU tests, and tests/golden/make_golden.py)."""
import math
import os

import torch

# Fixtures are stored as files of at most ~1 MB: a larger dict is split over <stem>.0.pt, <stem>.1.pt, ... by its top-level
# entries and, for dict / list entries (state_dict, grads, preds, cases, ...), by their items, in their original order.
FIXTURE_PART_BYTES = 800_000


def _nbytes(v):
    if torch.is_tensor(v):
        return v.numel() * v.element_size()
    if isinstance(v, dict):
        return sum(_nbytes(x) for x in v.values())
    if isinstance(v, (list, tuple)):
        return sum(_nbytes(x) for x in v)
    return 0


def save_fixture(obj, path):
    """torch.save(obj, path), or the parts <stem>.<i>.pt when obj holds more than FIXTURE_PART_BYTES of tensor data."""
    if _nbytes(obj) <= FIXTURE_PART_BYTES:
        torch.save(obj, path)
        return
    pieces = []                                          # (top-level key, sub key or None, value) in order
    for k, v in obj.items():
        if isinstance(v, dict) and _nbytes(v) > FIXTURE_PART_BYTES // 2:
            pieces += [(k, sk, sv) for sk, sv in v.items()]
        elif isinstance(v, list) and _nbytes(v) > FIXTURE_PART_BYTES // 2:
            pieces += [(k, i, sv) for i, sv in enumerate(v)]
        else:
            pieces.append((k, None, v))
    parts, cur, used = [], {}, 0
    for k, sk, v in pieces:
        n = _nbytes(v)
        if cur and used + n > FIXTURE_PART_BYTES:
            parts.append(cur)
            cur, used = {}, 0
        if sk is None:
            cur[k] = v
        elif isinstance(obj[k], list):
            cur.setdefault(k, []).append(v)
        else:
            cur.setdefault(k, {})[sk] = v
        used += n
    parts.append(cur)
    stem = path[:-3] if path.endswith(".pt") else path
    for i, part in enumerate(parts):
        torch.save(part, "%s.%d.pt" % (stem, i))


def load_fixture(golden_dir, name):
    """The fixture `name` of tests/golden, merged from its parts when it is stored split (see save_fixture)."""
    path = os.path.join(golden_dir, name)
    if os.path.exists(path):
        return torch.load(path, map_location="cpu", weights_only=False)
    stem = path[:-3] if path.endswith(".pt") else path
    out, i = {}, 0
    while os.path.exists("%s.%d.pt" % (stem, i)):
        for k, v in torch.load("%s.%d.pt" % (stem, i), map_location="cpu", weights_only=False).items():
            if isinstance(v, dict) and isinstance(out.get(k), dict):
                out[k].update(v)
            elif isinstance(v, list) and isinstance(out.get(k), list):
                out[k].extend(v)
            else:
                out[k] = v
        i += 1
    if i == 0:
        raise FileNotFoundError(path)
    return out


def formula_fill_(named_params):
    """Deterministic, RNG-free parameter values so large fixtures need not store weights.

    `named_params`: iterable of (name, tensor) — iterated in sorted-name order; frozen pos_emb tables are skipped."""
    with torch.no_grad():
        todo = sorted([(n, p) for n, p in named_params if not n.endswith("pos_emb")], key=lambda kv: kv[0])
        for i, (name, p) in enumerate(todo):
            idx = torch.arange(p.numel(), dtype=torch.float64)
            wave = torch.sin(idx * 0.37 + i * 1.3) + 0.5 * torch.cos(idx * 0.011 + i)
            if p.dim() >= 2:
                fan_in = p[0].numel()
                vals = wave * (0.7 / math.sqrt(fan_in))
            elif name.endswith("norm1.weight") or name.endswith("norm2.weight") or name.endswith("_norm.weight"):
                vals = 1.0 + 0.1 * wave
            else:
                vals = 0.05 * wave
            p.copy_(vals.reshape(p.shape).to(p.dtype))


def digest(t, n=256):
    """(l2 norm, n strided samples) of a tensor — compact stand-in for a full gradient in fixtures."""
    flat = t.detach().float().flatten()
    step = max(1, flat.numel() // n)
    return {"norm": flat.norm().clone(), "samples": flat[::step][:n].clone(), "step": step}


def rel_l2(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-12))
