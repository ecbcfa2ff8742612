// spark_types.h -- host-side rules for Spark's TimestampType and DecimalType: which source columns the engine takes and
// how it keeps them (source_type_of, used by decode_sources), and the exact comparison of scaled integers behind decimal
// literals (compare_scaled, used by the filter predicates).  Host code only; tests/native/spark_types.cu runs both.
#pragma once
#include <cstdint>

#include "hs_common.h"
#include "kernels.h"
#include "parquet_meta.h"

namespace hs {

// Spark types that ride on an int32 / int64 column (DevColumn::schema holds the leaf the index file declares)
inline bool is_decimal(const pq::SchemaColumn& s) { return s.converted_type == pq::CT_DECIMAL; }
inline bool is_timestamp(const pq::SchemaColumn& s) {
  return s.type == pq::INT64 && (s.converted_type == pq::CT_TIMESTAMP_MICROS || s.converted_type == pq::CT_TIMESTAMP_MILLIS);
}

// A source column as the engine keeps it: its HS storage type, how the decoder converts the stored values (ValueConv), and
// the Parquet leaf the index file declares for it.  Spark 3.1's TimestampType (INT96, INT64 TIMESTAMP_MILLIS / MICROS)
// becomes int64 micros, written as INT64 TIMESTAMP_MICROS; DecimalType(p <= 18) (INT32, INT64 or FIXED_LEN_BYTE_ARRAY)
// becomes its unscaled value, an int32 for p <= 9 and an int64 above, written as Spark writes it (INT32 / INT64 DECIMAL).
struct SourceType {
  int type;
  int conv;
  pq::SchemaColumn schema;
};

inline SourceType source_type_of(const pq::SchemaColumn& c, const char* file) {
  if (c.num_children > 0) fail(HS_EUNSUPPORTED, "%s: column '%s' is nested; only flat columns can be indexed", file, c.name.c_str());
  if (c.repetition == pq::REPEATED) fail(HS_EUNSUPPORTED, "%s: column '%s' is repeated", file, c.name.c_str());
  SourceType st{-1, CONV_NONE, c};
  st.schema.type_length = 0;
  st.schema.time_unit = 0;
  if (c.converted_type == pq::CT_DECIMAL && c.type == pq::BYTE_ARRAY)  // Spark: a decimal, hashed over its BigInteger bytes
    fail(HS_EUNSUPPORTED, "%s: column '%s' stores decimal(%d,%d) as BYTE_ARRAY; the GPU path handles INT32 / INT64 / "
         "FIXED_LEN_BYTE_ARRAY decimals", file, c.name.c_str(), c.precision, c.scale < 0 ? 0 : c.scale);
  if (c.converted_type == pq::CT_DECIMAL) {
    const int p = c.precision, s = c.scale < 0 ? 0 : c.scale;
    if (p > 18)
      fail(HS_EUNSUPPORTED, "%s: column '%s' is decimal(%d,%d); the GPU path handles decimal precision up to 18", file, c.name.c_str(), p, s);
    if (p < 1 || s > p) fail(HS_EFORMAT, "%s: column '%s' declares decimal(%d,%d)", file, c.name.c_str(), p, s);
    const bool narrow = p <= 9;
    if (c.type == pq::INT32) {
      if (!narrow) fail(HS_EFORMAT, "%s: column '%s' stores decimal(%d,%d) as INT32", file, c.name.c_str(), p, s);
    } else if (c.type == pq::INT64) {
      if (narrow) st.conv = CONV_NARROW;
    } else if (c.type == pq::FIXED_LEN_BYTE_ARRAY) {
      if (c.type_length < 1 || c.type_length > 16)
        fail(HS_EFORMAT, "%s: column '%s' is a decimal of %d bytes", file, c.name.c_str(), c.type_length);
      st.conv = CONV_FLBA;
    } else {
      fail(HS_EUNSUPPORTED, "%s: column '%s' stores a decimal as Parquet physical type %d", file, c.name.c_str(), c.type);
    }
    st.type = narrow ? HS_TYPE_INT32 : HS_TYPE_INT64;
    st.schema.type = narrow ? pq::INT32 : pq::INT64;
    st.schema.precision = p;
    st.schema.scale = s;
    return st;
  }
  if (c.type == pq::INT96 || (c.type == pq::INT64 && (c.converted_type == pq::CT_TIMESTAMP_MILLIS || c.time_unit == 1))) {
    st.conv = c.type == pq::INT96 ? CONV_INT96 : CONV_MILLIS;
    st.type = HS_TYPE_INT64;
    st.schema.type = pq::INT64;
    st.schema.converted_type = pq::CT_TIMESTAMP_MICROS;
    st.schema.precision = st.schema.scale = -1;
    return st;
  }
  if (c.type == pq::INT64 && c.time_unit == 3)
    fail(HS_EUNSUPPORTED, "%s: column '%s' is TIMESTAMP(NANOS), which Spark 3.1 does not read", file, c.name.c_str());
  switch (c.type) {
    case pq::BOOLEAN: st.type = HS_TYPE_BOOL; break;
    case pq::INT32: st.type = HS_TYPE_INT32; break;
    case pq::INT64: st.type = HS_TYPE_INT64; break;
    case pq::FLOAT: st.type = HS_TYPE_FLOAT; break;
    case pq::DOUBLE: st.type = HS_TYPE_DOUBLE; break;
    case pq::BYTE_ARRAY: st.type = HS_TYPE_STRING; break;  // Spark string / binary
    default:
      fail(HS_EUNSUPPORTED, "%s: column '%s' has Parquet physical type %d; the GPU path handles BOOLEAN/INT32/INT64/FLOAT/DOUBLE/BYTE_ARRAY",
           file, c.name.c_str(), c.type);
  }
  return st;
}

// a / 10^sa against b / 10^sb, exactly (Spark compares decimals, and integers with decimals, without rounding): the side
// with the larger scale is compared against the other scaled up, in 128 bits; past 10^19 a non-zero scaled value exceeds
// every int64, so its sign decides
inline int compare_scaled(int64_t a, int sa, int64_t b, int sb) {
  const bool up_b = sa > sb;  // scale b up by 10^k, else a
  const int k = up_b ? sa - sb : sb - sa;
  const int64_t x = up_b ? b : a, y = up_b ? a : b;  // x * 10^k against y
  int r;
  if (x == 0) r = 0 > y ? 1 : (0 < y ? -1 : 0);
  else if (k > 19) r = x > 0 ? 1 : -1;
  else {
    __int128 xs = x;
    for (int i = 0; i < k; i++) xs *= 10;
    r = xs > (__int128)y ? 1 : (xs < (__int128)y ? -1 : 0);
  }
  return up_b ? -r : r;  // r compares the scaled-up side with the other
}

}  // namespace hs
