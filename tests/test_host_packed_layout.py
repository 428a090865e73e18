"""The packed batch's header as the C header names it (the layout's specification) and as data.PackHeader
and ops describe it on the host: the same slot for every field, the same magic, header size and flag."""
import os
import re

import torch

from lanczosnetwork_b200 import data, ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _defines():
  with open(os.path.join(ROOT, 'include', 'lanczosnet_b200.h')) as fh:
    return {m.group(1): int(m.group(2), 0)
            for m in re.finditer(r'^#define (LNB_PACK\w*)\s+(0x[0-9a-fA-F]+|\d+)\b', fh.read(), re.M)}


def test_header_slots_match_pack_header():
  defs = _defines()
  slots = {name[len('LNB_PACK_HDR_'):]: v for name, v in defs.items()
           if name.startswith('LNB_PACK_HDR_') and name != 'LNB_PACK_HDR_BYTES'}
  fields = {f.upper(): f for f in data.PackHeader._fields}
  assert set(slots) == set(fields), set(slots) ^ set(fields)
  for name, slot in slots.items():
    assert slot == data.PackHeader._fields.index(fields[name]), name
  assert 4 * len(data.PackHeader._fields) <= defs['LNB_PACK_HDR_BYTES'] == 64


def test_magic_and_host_tiles_flag_match():
  defs = _defines()
  assert defs['LNB_PACK_MAGIC'] == data.PACK_MAGIC
  assert defs['LNB_PACKED_HOST_TILES'] == ops.PACKED_HOST_TILES


def test_packed_layout_is_the_header_pack_sparse_writes():
  samples = data.synthetic_qm8_samples(9, seed=4)
  for eigs in (False, True):
    sp = data.sparse_collate(samples, 20, eigs=eigs)
    for label in (False, True):
      blob = data.pack_sparse(sp, label=label)['blob']
      P = sp['label'].shape[1] if label else 0
      h = data.packed_layout(9, 20, len(sp['node_feat']), len(sp['edges']), eigs, P)
      assert data.read_packed_header(blob) == h == data.read_packed_header(torch.from_numpy(blob))
      assert h.total == blob.size
      assert not blob[4 * len(h):64].any()
