// The host build of the JPEG decode (jpeg_core_host.cpp) as a program, for tests/test_jpeg_fuzz_host.py to run under
// -fsanitize=address,undefined on damaged files: a sanitizer needs its runtime loaded first, which a library opened by Python is not.
// stdin: records of [u64 size][file bytes].  stdout, per record: [i32 rc][i32 w][i32 h][i32 wide][w * h * 3 RGB bytes when rc == 0],
// with rc and wide as jc_decode_wide's (rc 0, -2 corrupt data, 1 refused by the parse); w, h are 0 when the parse refuses the file.
#include "jpeg_core_host.cpp"

#include <stdio.h>

int main()
{
    uint64_t size;
    while (fread(&size, sizeof(size), 1, stdin) == 1) {
        std::vector<uint8_t> file(size);
        if (size && fread(file.data(), 1, size, stdin) != size) return 3;
        int32_t head[4] = {0, 0, 0, 0};
        char why[256];
        std::vector<uint8_t> rgb;
        head[0] = jc_info(file.data(), size, head + 1, why, sizeof(why));
        if (head[0] == 0) {
            rgb.resize(3 * (size_t)head[1] * (size_t)head[2]);
            head[0] = jc_decode_wide(file.data(), size, rgb.data(), rgb.size(), head + 1, why, sizeof(why), head + 3);
        }
        fwrite(head, sizeof(head), 1, stdout);
        if (head[0] == 0) fwrite(rgb.data(), 1, rgb.size(), stdout);
    }
    return 0;
}
