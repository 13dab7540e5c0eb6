// Text forms of datetime.fromtimestamp(ts) from its naive wall-clock second count (no microseconds), shared by the scan
// kernels (str(datetime) predicates) and the record formatter (isoformat(): sep 'T'; strftime("%Y-%m-%d"): date_only).
#pragma once
#include <stdint.h>

namespace fei {

// "YYYY-MM-DD<sep>HH:MM:SS", or "YYYY-MM-DD" alone when date_only (civil-from-days, proleptic Gregorian), character k given to
// out(k, c); returns the length
template <class Out>
__device__ __forceinline__ uint32_t civil_text(int64_t wall, uint8_t sep, bool date_only, Out out) {
  int64_t days = wall / 86400; int64_t rem = wall % 86400;
  if (rem < 0) { rem += 86400; --days; }
  const int64_t z = days + 719468;
  const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
  const uint32_t doe = (uint32_t)(z - era * 146097);
  const uint32_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  int64_t y = (int64_t)yoe + era * 400;
  const uint32_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const uint32_t mp = (5 * doy + 2) / 153;
  const uint32_t d = doy - (153 * mp + 2) / 5 + 1;
  const uint32_t m = mp < 10 ? mp + 3 : mp - 9;
  if (m <= 2) ++y;
  const uint32_t hh = (uint32_t)(rem / 3600), mi = (uint32_t)(rem % 3600 / 60), ss = (uint32_t)(rem % 60);
  uint32_t yy = (uint32_t)(y < 0 ? 0 : y > 9999 ? 9999 : y);
  out(0, '0' + yy / 1000); out(1, '0' + yy / 100 % 10); out(2, '0' + yy / 10 % 10); out(3, '0' + yy % 10); out(4, '-');
  out(5, '0' + m / 10); out(6, '0' + m % 10); out(7, '-'); out(8, '0' + d / 10); out(9, '0' + d % 10);
  if (date_only) return 10;
  out(10, sep);
  out(11, '0' + hh / 10); out(12, '0' + hh % 10); out(13, ':'); out(14, '0' + mi / 10); out(15, '0' + mi % 10); out(16, ':');
  out(17, '0' + ss / 10); out(18, '0' + ss % 10);
  return 19;
}
// str(datetime): "YYYY-MM-DD HH:MM:SS"
__device__ __forceinline__ uint32_t format_datetime(int64_t wall, uint8_t* out) {
  return civil_text(wall, ' ', false, [&](int k, uint32_t c) { out[k] = (uint8_t)c; });
}

}  // namespace fei
