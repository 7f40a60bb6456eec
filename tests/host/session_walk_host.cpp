// CPU harness of the streaming reader's record walk (walk_records over read_block_prefix) and the writer's carry rule (batch_bytes_out),
// kanzi-go_b200/csrc/kz_common.cuh, for tests/test_session_walk_host.py.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../kanzi-go_b200/csrc/kz_common.cuh"

extern "C" {
// Walks the window bytes[0 .. n) from bit start. res = {count, status, ended, next_bit}.
uint32_t walk(const uint8_t* bytes, uint64_t n, uint64_t start, uint32_t max_records, uint64_t max_bits, uint64_t* bit_off, uint64_t* bits, int64_t* res) {
    std::vector<uint32_t> words(n / 4 + 4, 0);  // bits_at reads one word past the last touched bit
    memcpy(words.data(), bytes, n);
    const kz::WalkResult r = kz::walk_records(words.data(), start, 8 * n, max_records, max_bits, bit_off, bits);
    res[0] = r.count;
    res[1] = r.status;
    res[2] = r.ended;
    res[3] = (int64_t)r.next_bit;
    return r.count;
}

// A stream cut into batches of batch_bits[i] bits (the concatenation of all of them is `bits`): every batch but the first starts with
// the carry of the one before it, hands out batch_bytes_out() bytes and carries the rest. out receives the bytes handed out, in order.
uint64_t carry_commit(const uint8_t* bits, const uint64_t* batch_bits, uint32_t nbatches, uint8_t* out) {
    uint64_t pos = 0, written = 0;
    uint32_t carry_bits = 0;
    uint8_t carry = 0;
    for (uint32_t i = 0; i < nbatches; i++) {
        std::vector<uint8_t> buf((carry_bits + batch_bits[i]) / 8 + 8, 0);
        kz::BitWriter bw(buf.data());
        if (carry_bits) bw.write(carry >> (8 - carry_bits), carry_bits);
        for (uint64_t b = 0; b < batch_bits[i]; b++, pos++) bw.write((bits[pos >> 3] >> (7 - (pos & 7))) & 1, 1);
        const uint64_t total = bw.pos;
        const uint64_t give = kz::batch_bytes_out(total, i + 1 == nbatches, &carry_bits);
        memcpy(out + written, buf.data(), give);
        written += give;
        carry = give < buf.size() ? buf[give] : 0;
    }
    return written;
}
}
