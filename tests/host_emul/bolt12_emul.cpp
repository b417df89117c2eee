// tests/host_emul/bolt12_emul.cpp — TEST-ONLY host build of lightning_b200/csrc/bolt12.cuh (linked into libemul.so).
//
// Runs the parse, leaf, nonce, branch and sighash functions the k_b12_* kernels call, in the order the kernels combine
// them: fields in stream order, signature-range fields dropped, the tree reduced level by level (neighbours paired, an
// odd last node carried up).  What this cannot check is the warp orchestration itself (ballot compaction, lane striding);
// tests/test_gpu_bolt12.py does that on the device.
#include <vector>
#include "../../lightning_b200/csrc/bolt12.cuh"

static void words_to_bytes(u8* out, const u32 w[8]) {
    for (int i = 0; i < 8; i++) {
        out[4 * i] = (u8)(w[i] >> 24); out[4 * i + 1] = (u8)(w[i] >> 16);
        out[4 * i + 2] = (u8)(w[i] >> 8); out[4 * i + 3] = (u8)w[i];
    }
}

// Returns the stream's field count, or -1 where the device reports status -1.  root32 / sighash32: zeros for -1.
extern "C" long long emul_bolt12(const u8* stream, u32 len, const u8* sigtag, u32 sigtag_len, u8* root32, u8* sighash32) {
    for (int i = 0; i < 32; i++) root32[i] = sighash32[i] = 0;
    long long cnt = b12_count(stream, len);
    if (cnt < 0) return -1;
    std::vector<b12_field> rec((size_t)cnt);
    u32 pos = 0;
    for (long long j = 0; j < cnt; j++)
        if (!b12_next(stream, len, &pos, j == 0, j ? rec[j - 1].type : 0, &rec[j])) return -2;  // count and walk disagree
    b12_tags t;
    b12_make_tags(&t, sigtag, sigtag_len);
    u32 nm[8];
    b12_nonce_mid(nm, stream + rec[0].off, rec[0].len);
    std::vector<u32> node;
    for (const b12_field& f : rec) {
        if (b12_is_signature(f.type)) continue;
        u32 h[8];
        b12_leaf_pair(h, &t, nm, stream, f);
        node.insert(node.end(), h, h + 8);
    }
    size_t m = node.size() / 8;
    while (m > 1) {
        size_t up = (m + 1) / 2;
        for (size_t k = 0; k < up; k++) {
            u32 h[8];
            if (2 * k + 1 < m) b12_branch(h, t.branch, &node[16 * k], &node[16 * k + 8]);
            else for (int q = 0; q < 8; q++) h[q] = node[16 * k + q];
            for (int q = 0; q < 8; q++) node[8 * k + q] = h[q];
        }
        m = up;
    }
    u32 root[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (m) for (int q = 0; q < 8; q++) root[q] = node[q];
    words_to_bytes(root32, root);
    b12_sighash(sighash32, &t, root);
    return cnt;
}
