// Test-infrastructure stand-in for <boost/align/aligned_allocator.hpp> (Boost is not installed in
// this image). Only what src/core/models/pairhmm/simd_pair_hmm.hpp:32 needs:
// an allocator template usable with std::vector that returns storage aligned for SIMD vectors.
#pragma once
#include <cstddef>
#include <cstdlib>
#include <new>

namespace boost { namespace alignment {

template <class T, std::size_t Alignment = 64>
class aligned_allocator
{
public:
    using value_type = T;
    template <class U> struct rebind { using other = aligned_allocator<U, Alignment>; };
    aligned_allocator() noexcept = default;
    template <class U> aligned_allocator(const aligned_allocator<U, Alignment>&) noexcept {}
    T* allocate(std::size_t n)
    {
        constexpr std::size_t a = Alignment < alignof(T) ? alignof(T) : (Alignment < sizeof(void*) ? sizeof(void*) : Alignment);
        void* p = nullptr;
        if (n == 0) n = 1;
        if (posix_memalign(&p, a, n * sizeof(T)) != 0) throw std::bad_alloc {};
        return static_cast<T*>(p);
    }
    void deallocate(T* p, std::size_t) noexcept { std::free(p); }
};

template <class T, class U, std::size_t A>
bool operator==(const aligned_allocator<T, A>&, const aligned_allocator<U, A>&) noexcept { return true; }
template <class T, class U, std::size_t A>
bool operator!=(const aligned_allocator<T, A>&, const aligned_allocator<U, A>&) noexcept { return false; }

}} // namespace boost::alignment
