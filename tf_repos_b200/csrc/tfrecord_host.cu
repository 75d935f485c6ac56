// tfrecord_host.cu -- HOST-side TFRecord framing behind the C ABI (no CUDA in this file).
//
// A TFRecord file is a chain of  uint64 length | uint32 masked_crc32c(length) | data | uint32 masked_crc32c(data)
// (tensorflow/core/lib/io/record_writer.cc).  Walking it is a serial chain of dependent 12-byte reads over a buffer the
// host has just read, so it stays on the host; the per-byte work (the data CRC, the protobuf) is done on the device
// (tfrecord_device.cu).  The checks and their order are those of tfrecord.read_records(verify_crc=True).
#include <string.h>

#include "common.cuh"

using namespace ctr;

namespace {

struct Crc32cTable {
  uint32_t t[256];
  Crc32cTable() {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0x82F63B78u : c >> 1;
      t[i] = c;
    }
  }
};

uint32_t crc32c(const uint8_t* p, size_t n) {
  static const Crc32cTable table;   // thread-safe one-time initialisation
  uint32_t c = 0xFFFFFFFFu;
  for (size_t i = 0; i < n; ++i) c = table.t[(c ^ p[i]) & 0xFF] ^ (c >> 8);
  return c ^ 0xFFFFFFFFu;
}

uint32_t masked_crc(const uint8_t* p, size_t n) {
  const uint32_t c = crc32c(p, n);
  return ((c >> 15) | (c << 17)) + 0xA282EAD8u;
}

uint64_t le64(const uint8_t* p) {
  uint64_t v;
  memcpy(&v, p, 8);
  return v;
}
uint32_t le32(const uint8_t* p) {
  uint32_t v;
  memcpy(&v, p, 4);
  return v;
}

// the device walks a record with int32 positions
constexpr uint64_t TFR_MAX_RECORD = 0x7FFFFFFFull - 16;

}  // namespace

extern "C" {

int ctr_tfrecord_frame(const void* buf_host, size_t len, int final_chunk, int64_t* rec_off, int64_t max_records,
                       int64_t* info) {
  if ((len && !buf_host) || max_records < 0 || (max_records && !rec_off) || !info) {
    set_error("ctr_tfrecord_frame: bad arguments");
    return CTR_ERR_INVALID_ARG;
  }
  const uint8_t* b = static_cast<const uint8_t*>(buf_host);
  int64_t n = 0, cls = CTR_TFR_OK, need = 12;
  size_t pos = 0;
  while (pos < len && n < max_records) {
    if (len - pos < 12) {
      if (final_chunk) cls = CTR_TFR_TRUNCATED_HEADER;
      break;
    }
    const uint64_t length = le64(b + pos);
    if (le32(b + pos + 8) != masked_crc(b + pos, 8)) { cls = CTR_TFR_CORRUPTED_LENGTH; break; }
    if (length > TFR_MAX_RECORD) { cls = CTR_TFR_TOO_LARGE; break; }
    need = 16 + (int64_t)length;
    if (len - pos < (size_t)need) {
      if (final_chunk) cls = CTR_TFR_TRUNCATED_RECORD;
      break;
    }
    rec_off[n++] = (int64_t)pos;
    pos += (size_t)need;
    need = 12;
  }
  info[0] = n;
  info[1] = (int64_t)pos;
  info[2] = cls;
  info[3] = (int64_t)pos;
  info[4] = need;
  return CTR_OK;
}

}  // extern "C"
