// Converts float32 bit patterns with the engine's observation conversions (bsb_obs_dtype.h), compiled on its own
// with a plain C++ compiler: tests/test_obs_dtype.py compares the results with torch.
//   convert <in.u32> <out_bf16.u16> <out_u8.u8>
#include <cstdio>
#include <vector>

#include "bsb_obs_dtype.h"

int main(int argc, char** argv) {
  if (argc != 4) { std::fprintf(stderr, "usage: convert in.u32 out.u16 out.u8\n"); return 2; }
  std::FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 1;
  std::vector<uint32_t> bits;
  uint32_t u;
  while (std::fread(&u, sizeof(u), 1, in) == 1) bits.push_back(u);
  std::fclose(in);
  std::vector<uint16_t> bf16;
  std::vector<uint8_t> u8;
  for (uint32_t b : bits) {
    float f;
    memcpy(&f, &b, sizeof(f));
    bf16.push_back(bsb::obs_cast<bsb::Bf16>(f).bits);
    u8.push_back(bsb::obs_cast<uint8_t>(f));
  }
  std::FILE* o16 = std::fopen(argv[2], "wb");
  std::FILE* o8 = std::fopen(argv[3], "wb");
  if (!o16 || !o8) return 1;
  std::fwrite(bf16.data(), sizeof(uint16_t), bf16.size(), o16);
  std::fwrite(u8.data(), sizeof(uint8_t), u8.size(), o8);
  std::fclose(o16);
  std::fclose(o8);
  std::printf("converted %zu\n", bits.size());
  return 0;
}
