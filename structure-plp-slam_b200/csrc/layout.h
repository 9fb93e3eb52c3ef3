// layout.h -- where the device buffers of one call or one handle live, and how host arrays get there.
//
// Each piece of device memory is declared once, against the pointer field that will hold its device address:
//   in(field, src, count)            `count` elements copied from host memory; a null src leaves the field null and takes
//                                    no bytes
//   in(field, src, count, capacity)  a piece of `capacity` elements whose first `count` are copied from src (src may be
//                                    null when count is 0); always placed, so the field is never null
//   out(field, count)                output / scratch space: neither copied nor cleared (it holds whatever the memory held;
//                                    every kernel writes its outputs before anything reads them)
//   same(field, of)                  `field` gets the address of the piece declared against `of`
// Every piece starts on a 256-byte boundary.  Inputs are placed first, in declaration order, then outputs, so one copy of
// in_bytes() bytes from the host image carries every input.  place() writes each field's device address BEFORE it copies
// any input into the host image: a job struct or table whose fields were declared here can itself be an input and rides
// in the same copy.  A declared field must therefore stay where it is until place(): a vector whose elements hold declared
// fields is sized before the first declaration.
//
// Host-only C++ (tests/test_layout.py compiles it with g++); the CUDA backings stage() / alloc() are in context.cu.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <type_traits>
#include <vector>

namespace plp {

class DevLayout {
  public:
    template <class T>
    void in(T *&field, const std::remove_const_t<T> *src, size_t count) {
        field = nullptr;
        if (src) in(field, src, count, count);
    }
    template <class T>
    void in(T *&field, const std::remove_const_t<T> *src, size_t count, size_t capacity) {
        ins_.push_back({&field, src, count * sizeof(T), capacity * sizeof(T)});
    }
    template <class T>
    void out(T *&field, size_t count) {
        outs_.push_back({&field, nullptr, 0, count * sizeof(T)});
    }
    // `field` gets the address of the piece declared against `of` (a buffer one job writes and another reads)
    template <class T, class U>
    void same(T *&field, U *const &of) {
        static_assert(std::is_convertible<U *, T *>::value, "incompatible pointer types");
        same_.push_back({&field, &of});
    }

    // bytes of the whole layout, and of the prefix that holds the inputs (the extent of the host-to-device copy)
    size_t bytes() const { return end(outs_, end(ins_, 0)); }
    size_t in_bytes() const {
        size_t off = 0, hi = 0;
        for (const Piece &p : ins_) {
            if (p.bytes && off + p.bytes > hi) hi = off + p.bytes;
            off += round(p.capacity);
        }
        return hi;
    }

    // Patches every field to its address under `dev`, then copies the inputs into the host image at the same offsets.
    // Returns in_bytes().
    size_t place(uint8_t *dev, uint8_t *host) {
        dev_ = dev;
        host_ = host;
        size_t off = 0;
        for (std::vector<Piece> *v : {&ins_, &outs_})
            for (Piece &p : *v) {
                p.off = off;
                void *addr = dev + off;
                memcpy(p.field, &addr, sizeof(addr));
                off += round(p.capacity);
            }
        for (const Alias &a : same_) memcpy(a.field, a.of, sizeof(void *));
        for (const Piece &p : ins_)
            if (p.bytes) memcpy(host + p.off, p.src, p.bytes);
        return in_bytes();
    }

    // the host-image address of a placed device address (outputs copied back into the image in one piece)
    template <class T>
    std::remove_const_t<T> *host(T *dev) const {
        return reinterpret_cast<std::remove_const_t<T> *>(host_ + (reinterpret_cast<const uint8_t *>(dev) - dev_));
    }

  private:
    struct Piece {
        void *field;  // the pointer field (T *) that receives the device address
        const void *src;
        size_t bytes, capacity;
        size_t off = 0;
    };
    static size_t round(size_t b) { return (b + 255) & ~(size_t)255; }
    static size_t end(const std::vector<Piece> &v, size_t off) {
        for (const Piece &p : v) off += round(p.capacity);
        return off;
    }
    struct Alias {
        void *field;
        const void *of;
    };
    std::vector<Piece> ins_, outs_;
    std::vector<Alias> same_;
    uint8_t *dev_ = nullptr, *host_ = nullptr;
};

}  // namespace plp
