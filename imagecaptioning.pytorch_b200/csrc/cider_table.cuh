// The CIDEr document-frequency table shared by the reward kernels (reward.cu) and the diversity kernels (diversity.cu): n-gram keys of
// token ids as array_to_str writes them (rewards.py:33-39), open addressing, idf = log(ref_len) - log(max(1, df)) per slot.
#pragma once

namespace capb200 {

constexpr int CIDER_MAXL = 64;        // max tokens in a caption incl. the closing 0 (diversity kernels; the rewards' short form)
constexpr int CIDER_MAXL_LONG = 256;  // the rewards' long form, for hypotheses or references past 64 tokens (= CAPB200_MAX_SEQ_LENGTH)
constexpr int CIDER_N = 4;

struct CiderSlot {
    int key[4];
    double idf;
};

struct CiderTable {
    CiderSlot* slots = nullptr;   // device, open addressing, key[0] == -2 marks an empty slot
    unsigned long long mask = 0;  // capacity - 1
    double log_ref_len = 0.0;
    long entries = 0;
    // corpus mode (CiderD(df='corpus'), ciderD_scorer.py:143-147,182-186,210-216): the slots are rebuilt on the device from the references of
    // every reward call; `used` [1] counts the occupied slots of the build under way
    bool corpus = false;
    unsigned int* used = nullptr;
};

__host__ __device__ inline unsigned long long cider_hash(int a, int b, int c, int d) {
    unsigned long long h = 0x9E3779B97F4A7C15ull;
    const int k[4] = {a, b, c, d};
    for (int i = 0; i < 4; ++i) {
        h ^= (unsigned long long)(unsigned int)k[i] + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
        h *= 0xBF58476D1CE4E5B9ull;
        h ^= h >> 31;
    }
    return h;
}

__device__ __forceinline__ bool same_gram(const int* a, const int* b, int n) {
    for (int i = 0; i < n; ++i) if (a[i] != b[i]) return false;
    return true;
}

__device__ __forceinline__ double cider_idf(const CiderSlot* __restrict__ slots, unsigned long long mask, double log_ref_len, const int* tok, int n) {
    const int k0 = tok[0], k1 = n > 1 ? tok[1] : -1, k2 = n > 2 ? tok[2] : -1, k3 = n > 3 ? tok[3] : -1;
    unsigned long long h = cider_hash(k0, k1, k2, k3) & mask;
    for (;;) {
        const CiderSlot& s = slots[h];
        if (s.key[0] == -2) return log_ref_len;                 // unseen n-gram: df = 0 -> log(max(1, 0)) = 0
        if (s.key[0] == k0 && s.key[1] == k1 && s.key[2] == k2 && s.key[3] == k3) return s.idf;
        h = (h + 1) & mask;
    }
}

}  // namespace capb200
