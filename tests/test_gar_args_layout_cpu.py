"""`ops.gar.GarArgs` is the argument block of the fused aggregation kernels, passed by address to `agb_gar_fused` and
`agb_gar_phase_a`: a field out of place would hand the kernels another field's value. This test parses `struct GarArgs` out of
`native/op_gar/gar.cu` and compares its fields (names, order, element types, array lengths) with the ctypes mirror."""

import ctypes
import pathlib
import re

from aggregathor_b200.ops import gar as gar_ops

SOURCE = pathlib.Path(__file__).resolve().parent.parent / "aggregathor_b200" / "native" / "op_gar" / "gar.cu"
SCALARS = {"int": ctypes.c_int, "uint32_t": ctypes.c_uint32, "long long": ctypes.c_longlong, "unsigned long long": ctypes.c_ulonglong,
           "float": ctypes.c_float, "double": ctypes.c_double}


def _constants(source):
  return {name: int(value) for name, value in re.findall(r"constexpr int (\w+) = (\d+);", source)}


def _struct_fields(source):
  """[(name, ctypes element type, array length or None)] of `struct GarArgs`, in declaration order."""
  body = re.search(r"\nstruct GarArgs \{(.*?)\n\};", source, re.S).group(1)
  body = re.sub(r"//[^\n]*", "", body)
  constants = _constants(source)
  fields = []
  for declaration in filter(None, (d.strip() for d in body.split(";"))):
    match = re.fullmatch(r"((?:unsigned )?(?:long long|int|uint32_t|float|double|__nv_bfloat16))( const)?\s*(\*?)\s*(.+)", declaration, re.S)
    assert match is not None, declaration
    base, _, pointer, declarators = match.groups()
    kind = ctypes.c_ulonglong if pointer else SCALARS[base]   # device addresses
    for declarator in declarators.split(","):
      name, length = re.fullmatch(r"\s*(\w+)(?:\[(\w+)\])?\s*", declarator).groups()
      fields.append((name, kind, None if length is None else int(length) if length.isdigit() else constants[length]))
  return fields


def _mirror_fields(structure):
  fields = []
  for name, kind in structure._fields_:
    if issubclass(kind, ctypes.Array):
      fields.append((name, kind._type_, kind._length_))
    else:
      fields.append((name, kind, None))
  return fields


def test_ctypes_mirror_matches_the_struct():
  assert _mirror_fields(gar_ops.GarArgs) == _struct_fields(SOURCE.read_text())

